"""Tensor-core engines of the dense path: wgmma implicit-GEMM convolutions (csrc/dense_tc.cu) plus their
memory-bound companions (csrc/dense_misc.cu).  EngineTC: bf16 operands (fast, ~1e-2); EngineTCSplit: f16x3 split
operands (fp32-faithful, the parity mode).  Both run the same layer methods; a format is its activation layout (`alloc`,
`dims`), its C entry points (`suffix`) and its weight packing.  Same interface as detector.EngineF32."""
import ctypes

import torch

from . import _lib


def _valid(valid_hw, n, device):
    """per-image valid extents as the kernels read them: device int32 [n, 2] = (h, w), contiguous"""
    assert tuple(valid_hw.shape) == (n, 2) and valid_hw.dtype == torch.int32 and valid_hw.device == device, \
        "valid_hw must be an int32 [N,2] tensor on the detector's device"
    return valid_hw.contiguous()


class EngineTC:
    name = "bf16"
    act_dtype = torch.bfloat16
    suffix = "bf16"                                      # C-ABI entry points of this engine's activation format

    def __init__(self, device):
        self.device = device
        self.lib = _lib.lib()

    def _call(self, name, *args):
        """the C entry point name % suffix, looked up at call time (tests substitute entry points on the library)"""
        fn = name % self.suffix
        _lib.check(getattr(self.lib, fn)(*args), fn)

    # ------------------------------------------------------------------ weights
    def _tc(self, L, out16=False):
        if L.tc is None:
            w = L.w_raw                                              # [Cout, KH, KW, Cin] fp32 (unpadded Cin)
            cout, kh, kw, cin = w.shape
            cout_p = ((cout + 31) // 32) * 32
            cin_p = ((cin + 63) // 64) * 64                          # per tap: whole 64-channel K blocks, zero padded
            wp4 = torch.zeros((cout_p, kh, kw, cin_p), dtype=torch.float32)
            wp4[:cout, :, :, :cin] = w
            wp = wp4.reshape(cout_p, kh * kw * cin_p)
            L.tc = dict(w=wp.to(self.device, torch.bfloat16).contiguous(), cout_p=cout_p)
        return L.tc

    def _stem_tc(self, L):
        if L.tc is None:
            w = L.w_raw                                              # [64, 7, 7, 3]
            wp = torch.zeros((64, 192), dtype=torch.float32)
            wp[:, :147] = w.reshape(64, 147)
            L.tc = dict(w=wp.to(self.device, torch.bfloat16).contiguous(), cout_p=64)
        return L.tc

    @staticmethod
    def _s2d_weights(L):
        """conv1 weights for the space-to-depth form, fp32 [64][kh' 0..3][kw' 0..3][16] with ky = 2kh'+dy-o,
        kx = 2kw'+dx-o, channel (dy*2+dx)*3+c (zero where ky/kx fall outside the kernel, channels 12-15 zero).  o = 1 for
        ResNet's 7x7 / s2 / pad 3 conv1, o = 3 for HRNet's 3x3 / s2 / pad 1 conv1: both read image row 2(oy+kh'-2)+dy, so
        one 4x4 stride-1 convolution of the same space-to-depth input computes either, with the same output extent"""
        w = L.w_raw                                                  # [64, k, k, 3], k = 7 or 3
        k = w.shape[1]
        assert tuple(w.shape) in ((64, 7, 7, 3), (64, 3, 3, 3)), tuple(w.shape)
        o = 4 - k // 2
        wp = torch.zeros((64, 4, 4, 16), dtype=torch.float32)
        for khp in range(4):
            for dy in range(2):
                ky = 2 * khp + dy - o
                if not 0 <= ky < k:
                    continue
                for kwp in range(4):
                    for dx in range(2):
                        kx = 2 * kwp + dx - o
                        if not 0 <= kx < k:
                            continue
                        ch = (dy * 2 + dx) * 3
                        wp[:, khp, kwp, ch:ch + 3] = w[:, ky, kx, :]
        return wp

    def _stem_s2d_tc(self, L):
        if getattr(L, "tc_s2d", None) is None:
            L.tc_s2d = self._s2d_weights(L).reshape(64, 256).to(self.device, torch.bfloat16).contiguous()
        return L.tc_s2d

    def _stem_s2d_operands(self, L):
        """(weights, weight-scale arguments) of orp_stem_conv_s2d_*"""
        return self._stem_s2d_tc(L), ()

    @staticmethod
    def _wscale(tc):
        """the weight-scale argument of the f16x3 entry points (none in bf16)"""
        return ()

    @staticmethod
    def _group_weights(L):
        """a grouped conv2's weights (L.w_raw [width, 3, 3, gw]) in the layout of orp_b200_group.h: fp32 [width, 9, 64], the row
        of output channel co holding the gw weights of its group at that group's place inside co's 64-channel block, zeros
        elsewhere"""
        width, kh, kw, gw = L.w_raw.shape
        wp = torch.zeros((width, kh * kw, 64), dtype=torch.float32)
        c0 = (torch.arange(width) % 64) // gw * gw                  # first input channel of co's group inside its block
        rows = torch.arange(width)
        w = L.w_raw.reshape(width, kh * kw, gw)
        for k in range(gw):
            wp[rows, :, c0 + k] = w[:, :, k]
        return wp

    def _group_tc(self, L):
        if L.tc is None:
            L.tc = dict(w=self._group_weights(L).to(self.device, torch.bfloat16).contiguous())
        return L.tc

    # ------------------------------------------------------------------ layers
    def prepare_input(self, img_nchw):
        img = img_nchw.to(self.device, torch.float32).contiguous()
        assert img.shape[1] == 3
        return img                                                   # the stem kernel reads the NCHW image directly

    def stem(self, img, L, mode="s2d"):
        """conv1 + folded BN + ReLU.  mode "s2d" (default): space-to-depth copy of the image (1/12 of the im2col bytes)
        + a 4x4 stride-1 tensor-core convolution reading it through TMA; "im2col" (bf16 only, also taken for odd H or W):
        K=192 rows materialised in HBM + plain GEMM"""
        assert mode in ("s2d", "im2col"), mode
        n, _, h, w = img.shape
        st = _lib.current_stream_ptr()
        if mode == "s2d" and not (h % 2 or w % 2):
            xs = self._s2d_input(n, h, w)
            self._call("orp_stem_s2d_%s", _lib.ptr(img), n, h, w, _lib.ptr(xs), st)
            return self._stem_conv_s2d(xs, L, n, h, w)
        ho, wo = (h + 6 - 7) // 2 + 1, (w + 6 - 7) // 2 + 1
        y = torch.empty((n, ho, wo, 64), dtype=torch.bfloat16, device=self.device)
        cols = torch.empty((n, ho, wo, 192), dtype=torch.bfloat16, device=self.device)
        _lib.check(self.lib.orp_stem_im2col_bf16(_lib.ptr(img), n, h, w, _lib.ptr(cols), st), "orp_stem_im2col_bf16")
        self._launch([cols], [y], self._stem_tc(L), 64, 1, 1, 192, 1, 0, L.bias, True, False, False)
        return y

    def stem_u8(self, img_u8, L, norm_cfg, valid_hw=None):
        """conv1 + folded BN + ReLU from decoded uint8 HWC tiles [N,H,W,3]; Normalize (mean/std/to_rgb of the test
        pipeline) is applied inside the space-to-depth transform kernel, and so is the Pad that follows it when valid_hw
        (device int32 [N,2] per-image extents) is given: pixels outside enter as 0.0"""
        n, h, w, c = img_u8.shape
        assert c == 3 and img_u8.dtype == torch.uint8 and img_u8.is_contiguous() and h % 2 == 0 and w % 2 == 0
        st = _lib.current_stream_ptr()
        xs = self._s2d_input(n, h, w)
        mean = (ctypes.c_float * 3)(*norm_cfg["mean"])
        std = (ctypes.c_float * 3)(*norm_cfg["std"])
        to_rgb = int(bool(norm_cfg["to_rgb"]))
        if valid_hw is None:
            self._call("orp_stem_s2d_u8_%s", _lib.ptr(img_u8), n, h, w, mean, std, to_rgb, _lib.ptr(xs), st)
        else:
            self._call("orp_stem_s2d_u8_padded_%s", _lib.ptr(img_u8), n, h, w, mean, std, to_rgb,
                       _lib.ptr(_valid(valid_hw, n, self.device)), _lib.ptr(xs), st)
        return self._stem_conv_s2d(xs, L, n, h, w)

    def _s2d_input(self, n, h, w):
        """the space-to-depth stem input: bf16 [N,H/2+3,W/2+3,16], or in split form its hi and lo planes one after the
        other - in both formats the bytes of an activation tensor of that shape"""
        return self.alloc(n, h // 2 + 3, w // 2 + 3, 16)

    def _stem_conv_s2d(self, xs, L, n, h, w):
        ws, scale = self._stem_s2d_operands(L)
        y = self.alloc(n, h // 2, w // 2, 64)
        self._call("orp_stem_conv_s2d_%s", _lib.ptr(xs), n, h, w, _lib.ptr(ws), _lib.ptr(L.bias), *scale, 1,
                   _lib.ptr(y), _lib.current_stream_ptr())
        return y

    def _launch(self, xs, ys, tc, cout, kh, kw, cin, stride, pad, bias, relu, out_f32, deform, res=None, res32=None,
                offsets=None, stats=None, masks=None):
        n = len(xs)
        arr = (_lib.TcProblem * n)()
        for i in range(n):
            arr[i].x = xs[i].data_ptr()
            arr[i].N, arr[i].H, arr[i].W = xs[i].shape[0], xs[i].shape[1], xs[i].shape[2]
            arr[i].out = ys[i].data_ptr()
            arr[i].residual_bf16 = res[i].data_ptr() if res is not None else None
            arr[i].residual_f32 = res32[i].data_ptr() if res32 is not None else None
            arr[i].offset = offsets[i].data_ptr() if offsets is not None else None
            arr[i].gn_stats = stats[i].data_ptr() if stats is not None else None
            arr[i].mask = masks[i].data_ptr() if masks is not None else None
        self._call("orp_conv2d_%s", n, arr, _lib.ptr(tc["w"]), cout, tc["cout_p"], kh, kw, cin, stride, pad, _lib.ptr(bias),
                   *self._wscale(tc), int(relu), int(out_f32), int(deform), _lib.current_stream_ptr())

    @staticmethod
    def _ksplit(n, ho, wo, L, nprob, relu, residual, out_f32, residual_f32):
        """split-K factor for a launch whose tiling would leave most of the 132 SMs idle (3x3 layers on small maps)"""
        if nprob != 1 or L.kh * L.kw != 9 or residual is not None or residual_f32 is not None or out_f32 or relu == 2 or L.cout % 8:
            return 1
        mt = -(-(n * ho * wo) // 128)
        if mt * -(-L.cout // 64) > 66:           # the narrow-tile (BN = 64) launch already fills half the machine: no split-K
            return 1
        tiles = mt * -(-L.cout // 256)
        return 9 if tiles * 9 <= 2 * 132 else 3

    def _conv_splitk(self, x, y, tc, L, relu, ks, stats, f16x3):
        ws = torch.empty((ks, y.shape[0], y.shape[1], y.shape[2], L.cout), dtype=torch.float32, device=self.device)
        q = _lib.TcProblem()
        q.x, q.N, q.H, q.W, q.out = x.data_ptr(), x.shape[0], x.shape[1], x.shape[2], y.data_ptr()
        q.gn_stats = stats.data_ptr() if stats is not None else None
        rc = self.lib.orp_conv2d_tc_splitk(ctypes.byref(q), _lib.ptr(tc["w"]), L.cout, tc["cout_p"], L.kh, L.kw, L.w_raw.shape[3], L.stride,
                                           L.pad, _lib.ptr(L.bias), int(f16x3), int(tc.get("s", 0)), int(bool(relu)), ks, _lib.ptr(ws),
                                           _lib.current_stream_ptr())
        _lib.check(rc, "orp_conv2d_tc_splitk")

    def conv_multi(self, xs, L, relu=False, residual=None, out_f32=False, residual_f32=None, stats=None):
        """relu: False/True, or 2 for the exact-GELU epilogue (Swin MLP); stats: per-problem double [N,32,2] tensors
        (zeroed) that receive the GroupNorm statistics of the outputs"""
        tc = self._tc(L, out16=not out_f32)
        ys = []
        for x in xs:
            n, h, w, cin = self.dims(x)
            assert cin == L.w_raw.shape[3] and x.dtype == self.act_dtype
            ho = (h + 2 * L.pad - L.kh) // L.stride + 1
            wo = (w + 2 * L.pad - L.kw) // L.stride + 1
            ys.append(torch.empty((n, ho, wo, L.cout), dtype=torch.float32, device=self.device) if out_f32 else
                      self.alloc(n, ho, wo, L.cout))
        ks = self._ksplit(ys[0].shape[0], ys[0].shape[1], ys[0].shape[2], L, len(xs), relu, residual, out_f32, residual_f32)
        if ks > 1:
            self._conv_splitk(xs[0], ys[0], tc, L, relu, ks, None if stats is None else stats[0], self.suffix == "f16x3")
            return ys
        self._launch(xs, ys, tc, L.cout, L.kh, L.kw, L.w_raw.shape[3], L.stride, L.pad, L.bias, relu, out_f32, False,
                     res=residual, res32=residual_f32, stats=stats)
        return ys

    def conv(self, x, L, relu=False, residual=None, out_f32=False):
        return self.conv_multi([x], L, relu, None if residual is None else [residual], out_f32)[0]

    def gn_multi(self, xs, norm, relu=False, ups=None, stats=None):
        """GroupNorm(32, 256) (+ReLU, + nearest-upsampled top-down add) of several tensors sharing gamma / beta
        in one launch; stats: per-tensor double [N,32,2] sums (from the conv epilogue) or None to compute them"""
        st = _lib.current_stream_ptr()
        k = len(xs)
        if stats is None:
            stats = []
            for x in xs:
                n, h, w, c = self.dims(x)
                s = torch.zeros((n, 32, 2), dtype=torch.float64, device=self.device)
                self._call("orp_gn_stats_%s", _lib.ptr(x), n, h * w, c, 32, _lib.ptr(s), st)
                stats.append(s)
        ys = [torch.empty_like(x) for x in xs]
        arr = (_lib.GnProblem * k)()
        for i, x in enumerate(xs):
            assert self.dims(x)[3] == 256 and x.dtype == self.act_dtype
            arr[i].x = x.data_ptr()
            arr[i].N, arr[i].H, arr[i].W = x.shape[0], x.shape[1], x.shape[2]
            arr[i].stats = stats[i].data_ptr()
            arr[i].up_src = ups[i].data_ptr() if ups is not None and ups[i] is not None else None
            arr[i].y = ys[i].data_ptr()
        self._call("orp_gn_apply_%s_multi", k, arr, 256, 32, _lib.ptr(norm.gamma), _lib.ptr(norm.beta), 1e-5, int(relu), st)
        return ys

    def gn(self, x, norm, relu=False, up=None, stats=None):
        return self.gn_multi([x], norm, relu=relu, ups=[up], stats=None if stats is None else [stats])[0]

    def conv_gn(self, x, L, norm, relu=False, up=None):
        st = torch.zeros((x.shape[0], 32, 2), dtype=torch.float64, device=self.device)
        y = self.conv_multi([x], L, stats=[st])[0]                     # statistics come out of the conv epilogue
        return self.gn(y, norm, relu=relu, up=up, stats=st)

    def conv_gn_multi(self, xs, L, norm, relu=False):
        sts = torch.zeros((len(xs), xs[0].shape[0], 32, 2), dtype=torch.float64, device=self.device)
        ys = self.conv_multi(xs, L, stats=[sts[i] for i in range(len(xs))])
        return self.gn_multi(ys, norm, relu=relu, stats=[sts[i] for i in range(len(xs))])

    def maxpool(self, x):
        n, h, w, c = self.dims(x)
        y = self.alloc(n, (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1, c)
        self._call("orp_maxpool3x3s2_%s", _lib.ptr(x), n, h, w, c, _lib.ptr(y), _lib.current_stream_ptr())
        return y

    def deform_conv_multi(self, xs, offsets, L, relu=False, masks=None):
        tc = self._tc(L)
        ys = []
        for x in xs:
            n, h, w, _ = self.dims(x)
            ys.append(self.alloc(n, (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1, L.cout))
        self._launch(xs, ys, tc, L.cout, L.kh, L.kw, L.w_raw.shape[3], L.stride, L.pad, L.bias, relu, False, True,
                     offsets=offsets, masks=masks)
        return ys

    def deform_conv(self, x, offset, L, relu=False, mask=None):
        """DCNv1; DCNv2 when mask ([N,H,W,KH*KW] fp32) is given: the modulation is folded into the bilinear corner
        weights inside the tensor-core kernel's A-operand producers"""
        return self.deform_conv_multi([x], [offset], L, relu, masks=None if mask is None else [mask])[0]

    def group_conv(self, x, L, groups, relu=False):
        """ResNeXt's grouped 3x3 conv2 (L.w_raw: [width, 3, 3, width / groups]) + folded bn2 + ReLU, orp_group_conv2d_*"""
        tc = self._group_tc(L)
        n, h, w, width = self.dims(x)
        assert x.dtype == self.act_dtype and width == L.cout
        y = self.alloc(n, (h + 2 - 3) // L.stride + 1, (w + 2 - 3) // L.stride + 1, width)
        q = _lib.TcProblem()
        q.x, q.N, q.H, q.W, q.out = x.data_ptr(), n, h, w, y.data_ptr()
        self._call("orp_group_conv2d_%s", ctypes.byref(q), _lib.ptr(tc["w"]), width, groups, L.stride, _lib.ptr(L.bias),
                   *self._wscale(tc), int(relu), _lib.current_stream_ptr())
        return y

    def hr_fuse(self, base, srcs):
        """relu(base + sum_k nearest_up(srcs[k-1], 2^k)), orp_hr_fuse_*: one HRModule output branch (hrnet.py:182-190)"""
        n, h, w, c = self.dims(base)
        y = self.alloc(n, h, w, c)
        self._call("orp_hr_fuse_%s", _lib.ptr(base), n, h, w, c, len(srcs), _lib.ptr_array(srcs), _lib.ptr(y),
                   _lib.current_stream_ptr())
        return y

    def hrfpn_reduce(self, parts):
        """sum_i bilinear_up(parts[i], 2^i) of fp32 NHWC parts into this engine's format, orp_hrfpn_reduce_*"""
        n, h, w, c = parts[0].shape
        y = self.alloc(n, h, w, c)
        self._call("orp_hrfpn_reduce_%s", len(parts), _lib.ptr_array(parts), n, h, w, c, _lib.ptr(y), _lib.current_stream_ptr())
        return y

    def hrfpn_pool(self, x, max_pool):
        """avg / max pools of kernel = stride 2, 4, 8, 16 of x in one pass, orp_hrfpn_pool_*"""
        n, h, w, c = self.dims(x)
        outs = [self.alloc(n, h >> l, w >> l, c) for l in range(1, 5)]
        self._call("orp_hrfpn_pool_%s", _lib.ptr(x), n, h, w, c, int(bool(max_pool)), _lib.ptr_array(outs),
                   _lib.current_stream_ptr())
        return outs

    def to_float(self, x):
        """activation tensor of this engine -> fp32 NHWC"""
        return x.float()

    def from_float(self, x):
        return x.to(self.device, torch.bfloat16).contiguous()

    def alloc(self, b, h, w, c, zero=False):
        f = torch.zeros if zero else torch.empty
        return f((b, h, w, c), dtype=torch.bfloat16, device=self.device)

    @staticmethod
    def dims(x):
        """(B, H, W, C) of an activation tensor of this engine"""
        return tuple(x.shape)


class EngineTCSplit(EngineTC):
    """f16x3 arithmetic on the same wgmma kernels - the PARITY mode (include/orp_b200.h, "split" section): every fp32
    value is an fp16 pair hi + lo, every product hi*hi + lo*hi + hi*lo in one fp32 accumulator.  Activations are
    fp16 tensors [N,H,W,2,C] (hi channels, then lo channels)."""
    name = "f16x3"
    act_dtype = torch.float16
    suffix = "f16x3"

    @staticmethod
    def _split_weights(wp):
        """fp32 [..] -> (hi, lo, s): fp16 halves of w * 2^s, s in 0..15 chosen so the scaled weights have rms ~ 1 (keeps
        the lo halves in the normal fp16 range without risking overflow of the hi halves)"""
        nz = wp[wp != 0]
        s = 0
        if nz.numel():
            rms = float(nz.double().pow(2).mean().sqrt())
            amax = float(nz.abs().max())
            s = int(max(0, min(15, round(-float(torch.log2(torch.tensor(rms)))))))
            while s > 0 and amax * (2.0 ** s) > 16384.0:
                s -= 1
        ws = wp.double() * (2.0 ** s)
        hi = ws.to(torch.float16)
        lo = (ws - hi.double()).to(torch.float16)
        return hi, lo, s

    @staticmethod
    def _pad_cout(cout):
        """weight rows = output columns the kernel computes: a multiple of 64 (TMA-store tiles; the store clips at Cout), 32 for the
        small fp32 heads.  The kernel takes the widest accumulator (<= 256) that divides the padded count; 129..256 channels are
        padded to ONE 256-wide tile (Swin's 192-channel proj / fc2 / reduction layers: 3 x BN 64 -> 1 x BN 256, measured 279 -> 174 us
        at K = 768, 92 -> 77 us at K = 192).  Padding the other odd widths up to wider tiles (288 -> 384, 576 -> 640, 1152 -> 1280)
        was measured neutral to 10 % slower - those layers are bound by their epilogue / stores, not by MMA issue."""
        if cout <= 32:
            return ((cout + 31) // 32) * 32
        if 128 < cout <= 256:
            return 256
        return ((cout + 63) // 64) * 64

    def _tc(self, L, out16=False):
        """out16: the layer writes 16-bit outputs, whose TMA epilogue needs at least one 64-column tile (HRNet's 24- and
        32-channel branches); the 32-row padding serves the narrow fp32 outputs only"""
        if getattr(L, "tc3", None) is None:
            w = L.w_raw                                              # [Cout, KH, KW, Cin] fp32 (unpadded Cin)
            cout, kh, kw, cin = w.shape
            cout_p = 64 if out16 and cout <= 32 else self._pad_cout(cout)
            cin_p = ((cin + 63) // 64) * 64
            wp4 = torch.zeros((cout_p, kh * kw, cin_p), dtype=torch.float32)
            wp4[:cout, :, :cin] = w.reshape(cout, kh * kw, cin)
            hi, lo, s = self._split_weights(wp4)
            cbn = cin_p // 64                                        # [cout_p, taps, channel block, (hi, lo), 64]: the two halves
            wp = torch.stack([hi.reshape(cout_p, kh * kw, cbn, 64), lo.reshape(cout_p, kh * kw, cbn, 64)], dim=3)   # of a block are adjacent
            L.tc3 = dict(w=wp.reshape(cout_p, -1).to(self.device).contiguous(), cout_p=cout_p, s=s)
        return L.tc3

    def _group_tc(self, L):
        if getattr(L, "tc3", None) is None:
            hi, lo, s = self._split_weights(self._group_weights(L))    # [width, 9 taps, (hi, lo), 64]
            L.tc3 = dict(w=torch.stack([hi, lo], dim=2).reshape(L.cout, -1).to(self.device).contiguous(), s=s)
        return L.tc3

    def _stem_s2d_tc(self, L):
        if getattr(L, "tc3_s2d", None) is None:
            hi, lo, s = self._split_weights(self._s2d_weights(L).reshape(64, 4, 64))   # taps = kh', 64 virtual channels = (kw', 16)
            L.tc3_s2d = dict(w=torch.stack([hi, lo], dim=2).reshape(64, -1).to(self.device).contiguous(), s=s)
        return L.tc3_s2d

    def _stem_s2d_operands(self, L):
        ws = self._stem_s2d_tc(L)
        return ws["w"], (ws["s"],)

    @staticmethod
    def _wscale(tc):
        return (tc["s"],)

    # the same launch as the class attribute of this engine: patching one engine class's _launch (as tests do to record
    # which kernel a layer reaches) leaves the other's alone
    _launch = EngineTC._launch

    def stem(self, img, L, mode="s2d"):
        assert img.shape[2] % 2 == 0 and img.shape[3] % 2 == 0 and mode == "s2d", \
            "the f16x3 stem runs in space-to-depth form (even H, W)"
        return super().stem(img, L, mode)

    def to_float(self, x):
        n, h, w, c = self.dims(x)
        y = torch.empty((n, h, w, c), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.orp_split_to_f32(_lib.ptr(x), n * h * w, c, _lib.ptr(y), _lib.current_stream_ptr()), "orp_split_to_f32")
        return y

    def from_float(self, x):
        x = x.to(self.device, torch.float32).contiguous()
        n, h, w, c = x.shape
        y = self.alloc(n, h, w, c)
        _lib.check(self.lib.orp_split_from_f32(_lib.ptr(x), n * h * w, c, _lib.ptr(y), _lib.current_stream_ptr()), "orp_split_from_f32")
        return y

    def alloc(self, b, h, w, c, zero=False):
        f = torch.zeros if zero else torch.empty
        return f((b, h, w, 2, c), dtype=torch.float16, device=self.device)

    @staticmethod
    def dims(x):
        b, h, w, two, c = x.shape
        assert two == 2, "split activations are [N,H,W,2,C]"
        return b, h, w, c

    def overflow_count(self, reset=True):
        """saturated f16x3 stores since the last reset, after every launch enqueued so far on the current stream (waits
        for them).  The counter is one per process: it also holds what other engines, threads and streams recorded"""
        c = ctypes.c_uint(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.orp_f16x3_overflow_count(ctypes.byref(c), int(reset), _lib.current_stream_ptr()),
                       "orp_f16x3_overflow_count")
        return int(c.value)
