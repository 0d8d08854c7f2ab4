"""HRNet backbones (mmdet/models/backbones/hrnet.py) with the HRFPN neck (necks/hrfpn.py) on the liborp_b200 engines.

`HRNetArch` describes a backbone as the reference's `extra` dict does; `ARCHS` names the published HRNetV2p widths.
`HRNetGraph` runs backbone + HRFPN on one engine (detector.EngineF32 or engine_tc.EngineTC / EngineTCSplit):
- every convolution is the engine's convolution with the eval-mode BN folded in, ReLU and residual in its epilogue;
- every branch is carried at its width rounded up to a multiple of 8 (HRNetV2p-W18: 18 -> 24, 36 -> 40), with zero weight
  rows and zero biases in the pad channels: they stay exactly 0 through every layer, and later layers read zero weight
  columns there, so the real channels are those of the unpadded network;
- an HRModule's output branch i (hrnet.py:182-190) is: x_i plus each lower branch's stride-2 chain, the last conv of each
  chain adding the running sum in its residual epilogue; then one orp_hr_fuse launch adds the 1x1 + BN terms of the
  higher branches, nearest-upsampled, and applies the ReLU (the lowest-resolution branch has none: its last chain conv
  applies it);
- HRFPN's reduction_conv is applied before the upsampling: a 1x1 convolution and bilinear interpolation commute, so
  W cat(up_i(x_i)) + b = sum_i up_i(W_i x_i) + b with W_i the column slice of branch i.  The slices run at branch resolution
  with fp32 outputs, and orp_hrfpn_reduce sums them upsampled; the 480..720-channel concatenation never exists;
- orp_hrfpn_pool writes the four pooled levels from one read of the reduced map; the fpn_convs are the engine's
  convolutions with bias (HRFPN's ConvModules have no norm: hrfpn.py:49-66 never passes norm_cfg on)."""
from dataclasses import dataclass

import torch

from .weights import fold_bn

BLOCK_EXPANSION = {'BASIC': 1, 'BOTTLENECK': 4}


@dataclass(frozen=True)
class HRStage:
    num_modules: int
    block: str
    num_blocks: tuple
    num_channels: tuple

    @property
    def num_branches(self):
        return len(self.num_channels)

    @property
    def widths(self):
        """the branches' output widths (num_channels times the block's expansion)"""
        return tuple(c * BLOCK_EXPANSION[self.block] for c in self.num_channels)


@dataclass(frozen=True)
class HRNetArch:
    name: str
    stages: tuple                      # four HRStage: stage1 (layer1) .. stage4

    @classmethod
    def from_extra(cls, extra, name="hrnet"):
        """the architecture of HRNet(extra); ValueError where the reference's own checks fail (_check_branches),
        NotImplementedError for what the engine does not build (stages of other than 1, 2, 3, 4 branches, BOTTLENECK
        blocks in stages 2-4)"""
        stages = []
        for s in range(1, 5):
            cfg = extra['stage%d' % s]
            nb, blocks, chans = cfg['num_branches'], tuple(cfg['num_blocks']), tuple(cfg['num_channels'])
            if nb != len(blocks) or nb != len(chans):
                raise ValueError("stage%d: NUM_BRANCHES(%d) <> NUM_BLOCKS(%d) / NUM_CHANNELS(%d)" % (s, nb, len(blocks), len(chans)))
            if nb != s:
                raise NotImplementedError("stage%d has num_branches=%d: liborp_b200 builds HRNets whose stages 1-4 have 1, 2, 3 "
                                          "and 4 branches" % (s, nb))
            if cfg['block'] not in BLOCK_EXPANSION:
                raise ValueError("stage%d: block %r is not 'BASIC' or 'BOTTLENECK'" % (s, cfg['block']))
            if s > 1 and cfg['block'] != 'BASIC':
                raise NotImplementedError("stage%d: block=%r: liborp_b200 builds BASIC blocks in HRNet stages 2-4"
                                          % (s, cfg['block']))
            if cfg['num_modules'] < 1 or any(b < 1 for b in blocks) or any(c < 1 for c in chans):
                raise ValueError("stage%d: num_modules, num_blocks and num_channels must be positive" % s)
            stages.append(HRStage(int(cfg['num_modules']), cfg['block'], blocks, chans))
        for a in ARCHS.values():                   # a published architecture keeps its name
            if a.stages == tuple(stages):
                return a
        return cls(name, tuple(stages))

    def extra(self):
        return {'stage%d' % (s + 1): dict(num_modules=st.num_modules, num_branches=st.num_branches, block=st.block,
                                           num_blocks=st.num_blocks, num_channels=st.num_channels)
                for s, st in enumerate(self.stages)}

    @property
    def out_widths(self):
        """the widths of the four stage-4 outputs: HRFPN's in_channels"""
        return self.stages[3].widths


def _v2p(w):
    return HRNetArch("hrnetv2p_w%d" % w, (HRStage(1, 'BOTTLENECK', (4,), (64,)), HRStage(1, 'BASIC', (4, 4), (w, 2 * w)),
                                         HRStage(4, 'BASIC', (4, 4, 4), (w, 2 * w, 4 * w)),
                                         HRStage(3, 'BASIC', (4, 4, 4, 4), (w, 2 * w, 4 * w, 8 * w))))


# the published HRNetV2p backbones (configs/hrnet/*.py of mmdetection)
ARCHS = {a.name: a for a in (_v2p(18), _v2p(32), _v2p(40), _v2p(48))}


def arch_of(depth):
    """the HRNetArch the detector's `depth` names (a key of ARCHS, or an HRNetArch), None for another backbone"""
    if isinstance(depth, HRNetArch):
        return depth
    if isinstance(depth, str) and depth in ARCHS:
        return ARCHS[depth]
    return None


def pad8(c):
    return (c + 7) // 8 * 8


def transition_convs(pre, cur):
    """_make_transition_layer (hrnet.py:352-396): per new branch i, None or the list of (key suffix, cout, cin, stride) of
    its conv + BN + ReLU layers"""
    out = []
    for i in range(len(cur)):
        if i < len(pre):
            out.append(None if cur[i] == pre[i] else [("%d.0" % i, "%d.1" % i, cur[i], pre[i], 1)])
        else:
            chain = []
            for j in range(i + 1 - len(pre)):
                cout = cur[i] if j == i - len(pre) else pre[-1]
                chain.append(("%d.%d.0" % (i, j), "%d.%d.1" % (i, j), cout, pre[-1], 2))
            out.append(chain)
    return out


def fuse_convs(widths):
    """_make_fuse_layers (hrnet.py:113-173): [i][j] = None (j == i), or the list of (conv key, bn key, cout, cin, k, stride)
    of the path from branch j to output branch i"""
    nb = len(widths)
    out = []
    for i in range(nb):
        row = []
        for j in range(nb):
            if j > i:
                row.append([("%d.%d.0" % (i, j), "%d.%d.1" % (i, j), widths[i], widths[j], 1, 1)])
            elif j == i:
                row.append(None)
            else:
                row.append([("%d.%d.%d.0" % (i, j, k), "%d.%d.%d.1" % (i, j, k), widths[i] if k == i - j - 1 else widths[j],
                             widths[j], 3, 2) for k in range(i - j)])
        out.append(row)
    return out


def backbone_convs(arch):
    """every conv + BN pair of HRNet(arch.extra()) in a fixed order: (conv key, bn key, cout, cin, k, last_norm), keys
    without the 'backbone.' prefix; last_norm marks a residual block's last BN (the one zero_init_residual zeroes)"""
    out = [("conv1", "bn1", 64, 3, 3, False), ("conv2", "bn2", 64, 64, 3, False)]
    s1 = arch.stages[0]
    ch, inpl = s1.num_channels[0], 64
    for b in range(s1.num_blocks[0]):
        p = "layer1.%d." % b
        if s1.block == 'BOTTLENECK':
            out += [(p + "conv1", p + "bn1", ch, inpl, 1, False), (p + "conv2", p + "bn2", ch, ch, 3, False),
                    (p + "conv3", p + "bn3", ch * 4, ch, 1, True)]
        else:
            out += [(p + "conv1", p + "bn1", ch, inpl, 3, False), (p + "conv2", p + "bn2", ch, ch, 3, True)]
        if b == 0 and inpl != s1.widths[0]:
            out.append((p + "downsample.0", p + "downsample.1", s1.widths[0], inpl, 1, False))
        inpl = s1.widths[0]
    pre = s1.widths
    for s in range(1, 4):
        st = arch.stages[s]
        for t in transition_convs(pre, st.widths):
            for ck, bk, cout, cin, _ in t or ():
                out.append(("transition%d.%s" % (s, ck), "transition%d.%s" % (s, bk), cout, cin, 3, False))
        for m in range(st.num_modules):
            p = "stage%d.%d." % (s + 1, m)
            for br, (nblk, c) in enumerate(zip(st.num_blocks, st.widths)):
                for k in range(nblk):
                    q = p + "branches.%d.%d." % (br, k)
                    out += [(q + "conv1", q + "bn1", c, c, 3, False), (q + "conv2", q + "bn2", c, c, 3, True)]
            for row in fuse_convs(st.widths):
                for path in row:
                    for ck, bk, cout, cin, k, _ in path or ():
                        out.append((p + "fuse_layers." + ck, p + "fuse_layers." + bk, cout, cin, k, False))
        pre = st.widths
    return out


class HRNetGraph:
    """HRNet (from conv2 on) + HRFPN(stride 2, 5 outputs) on an engine; the stem's conv1 runs in the detector, on the
    stem kernels of a ResNet's conv1 (EngineTC._s2d_weights)"""

    def __init__(self, sd, device, eng, arch, pooling_type='AVG'):
        from .detector import ConvLayer
        self.eng, self.arch, self.max_pool = eng, arch, pooling_type == 'MAX'
        shapes = {ck: (cout, cin, k) for ck, _, cout, cin, k, _ in backbone_convs(arch)}

        def folded(conv, bn, stride, pad, cin_p=None):
            """conv + BN of the backbone, folded, rows and columns zero-padded to multiples of 8"""
            cout, cin, k = shapes[conv]
            w, b = sd["backbone." + conv + ".weight"], "backbone." + bn
            if tuple(w.shape) != (cout, cin, k, k):
                raise ValueError("backbone.%s.weight has shape %s where %s needs %s" % (conv, tuple(w.shape), arch.name, (cout, cin, k, k)))
            w, bias = fold_bn(w.float(), sd[b + ".weight"].float(), sd[b + ".bias"].float(), sd[b + ".running_mean"].float(),
                              sd[b + ".running_var"].float())
            cin_p = pad8(cin) if cin_p is None else cin_p
            wp = torch.zeros(pad8(cout), cin_p, k, k)
            wp[:cout, :cin] = w
            bp = torch.zeros(pad8(cout))
            bp[:cout] = bias
            return ConvLayer(wp, bp, stride, pad, device)

        self.conv2 = folded("conv2", "bn2", 2, 1)
        s1 = arch.stages[0]
        self.layer1 = []
        for b in range(s1.num_blocks[0]):
            p = "layer1.%d." % b
            blk = dict(ds=folded(p + "downsample.0", p + "downsample.1", 1, 0) if p + "downsample.0" in shapes else None)
            if s1.block == 'BOTTLENECK':
                blk["convs"] = [folded(p + "conv1", p + "bn1", 1, 0), folded(p + "conv2", p + "bn2", 1, 1),
                                folded(p + "conv3", p + "bn3", 1, 0)]
            else:
                blk["convs"] = [folded(p + "conv1", p + "bn1", 1, 1), folded(p + "conv2", p + "bn2", 1, 1)]
            self.layer1.append(blk)
        self.transitions, self.stages = [], []
        pre = s1.widths
        for s in range(1, 4):
            st = arch.stages[s]
            self.transitions.append([None if t is None else
                                     [folded("transition%d.%s" % (s, ck), "transition%d.%s" % (s, bk), stride, 1)
                                      for ck, bk, _, _, stride in t] for t in transition_convs(pre, st.widths)])
            mods = []
            for m in range(st.num_modules):
                p = "stage%d.%d." % (s + 1, m)
                branches = [[[folded(p + "branches.%d.%d.conv%d" % (br, k, c), p + "branches.%d.%d.bn%d" % (br, k, c), 1, 1)
                              for c in (1, 2)] for k in range(nblk)] for br, nblk in enumerate(st.num_blocks)]
                fuse = [[None if path is None else
                         [folded(p + "fuse_layers." + ck, p + "fuse_layers." + bk, stride, k // 2) for ck, bk, _, _, k, stride in path]
                         for path in row] for row in fuse_convs(st.widths)]
                mods.append((branches, fuse))
            self.stages.append(mods)
            pre = st.widths
        # HRFPN: reduction_conv column slices per branch (bias on branch 0), fpn_convs 3x3 / s2 with bias
        widths = arch.out_widths
        red = sd["neck.reduction_conv.conv.weight"].float()
        if tuple(red.shape[1:]) != (sum(widths), 1, 1) or tuple(sd["neck.reduction_conv.conv.bias"].shape) != (red.shape[0],):
            raise ValueError("neck.reduction_conv.conv.weight %s: HRFPN's in_channels must be the stage-4 widths %s of %s"
                             % (tuple(red.shape), list(widths), arch.name))
        self.out_channels = red.shape[0]
        self.reduce, c0 = [], 0
        for i, c in enumerate(widths):
            wp = torch.zeros(self.out_channels, pad8(c), 1, 1)
            wp[:, :c] = red[:, c0:c0 + c]
            c0 += c
            self.reduce.append(ConvLayer(wp, sd["neck.reduction_conv.conv.bias"].float() if i == 0 else None, 1, 0, device))
        self.fpn = [ConvLayer(sd["neck.fpn_convs.%d.conv.weight" % i].float(), sd["neck.fpn_convs.%d.conv.bias" % i].float(),
                              2, 1, device) for i in range(5)]

    def _conv_chain(self, x, chain, last_relu=True, residual=None):
        for L in chain[:-1]:
            x = self.eng.conv(x, L, relu=True)
        return self.eng.conv(x, chain[-1], relu=last_relu, residual=residual)

    def _fuse(self, xs, fuse):
        e, nb = self.eng, len(xs)
        out = []
        for i in range(nb):
            base = xs[i]
            for j in range(i):                  # stride-2 chains of the lower branches, each adding the running sum
                base = self._conv_chain(xs[j], fuse[i][j], last_relu=(i == nb - 1 and j == i - 1), residual=base)
            if i == nb - 1:
                out.append(base)
            else:
                out.append(e.hr_fuse(base, [e.conv(xs[j], fuse[i][j][0]) for j in range(i + 1, nb)]))
        return out

    def backbone(self, x):
        """x: the stem's conv1 output (after its BN and ReLU) -> the four stage-4 branches, channel-padded"""
        e = self.eng
        x = e.conv(x, self.conv2, relu=True)
        for blk in self.layer1:
            idt = x if blk["ds"] is None else e.conv(x, blk["ds"])
            for L in blk["convs"][:-1]:
                x = e.conv(x, L, relu=True)
            x = e.conv(x, blk["convs"][-1], relu=True, residual=idt)
        xs = [x]
        for trans, mods in zip(self.transitions, self.stages):
            # hrnet.py:492-513: a new branch, or a changed width, is made from the last branch of the previous stage
            xs = [xs[i] if t is None else self._conv_chain(xs[-1], t) for i, t in enumerate(trans)]
            for branches, fuse in mods:
                new = []
                for x, blocks in zip(xs, branches):
                    for c1, c2 in blocks:
                        x = e.conv(e.conv(x, c1, relu=True), c2, relu=True, residual=x)
                    new.append(x)
                xs = self._fuse(new, fuse)
        return xs

    def neck(self, xs):
        """HRFPN (hrfpn.py:78-100, stride 2): the five levels at strides 8 .. 128"""
        e = self.eng
        parts = [e.conv(x, L, out_f32=True) for x, L in zip(xs, self.reduce)]
        red = e.hrfpn_reduce(parts)
        levels = [red] + e.hrfpn_pool(red, self.max_pool)
        return [e.conv(x, L) for x, L in zip(levels, self.fpn)]
