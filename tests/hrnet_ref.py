"""fp64 evaluation of the dense graph with an HRNet backbone and the HRFPN neck (test infrastructure): hrnet.py / hrfpn.py
restated with F.conv2d and the eval-mode BN of oracle/torch_reference.py, with that file's head.  Two switches restate the
engine's rewrites of the graph, so that each can be checked against the reference's own modules on the CPU:
- `padded`: every branch carried at its width rounded up to a multiple of 8, zero weight rows / columns and zero BN
  shift in the pad channels (the pad channels stay 0 and are dropped at the end);
- `engine_order`: an HRModule's output branch summed as the engine sums it (x_i, then each lower branch's chain, then the
  upsampled higher branches), and HRFPN's 1x1 reduction applied per branch before the bilinear upsampling."""
import torch
import torch.nn.functional as F

from oracle import torch_reference as tr
from orientedreppoints_b200.hrnet import ARCHS, fuse_convs, pad8, transition_convs

# the batches the HRNet launches are tested at: one 1024 tile, the benchmark's 16 tiles, two 512 tiles; 960 (a 240 map)
BATCHES = [(1, 1024), (16, 1024), (2, 512), (1, 960)]


class _Params:
    """conv weight + BN of the state dict, optionally channel-padded"""

    def __init__(self, sd, padded):
        self.sd, self.padded = sd, padded

    def conv_bn(self, x, conv, bn, stride, relu=False, residual=None):
        w = self.sd["backbone." + conv + ".weight"]
        p = "backbone." + bn
        g, b, m, v = (self.sd[p + s] for s in (".weight", ".bias", ".running_mean", ".running_var"))
        if self.padded:
            co, ci = pad8(w.shape[0]), x.shape[1]
            wp = w.new_zeros(co, ci, *w.shape[2:])
            wp[:w.shape[0], :w.shape[1]] = w
            g, b, m, v = [torch.cat([t, t.new_full((co - t.shape[0],), fill)]) for t, fill in ((g, 0.), (b, 0.), (m, 0.), (v, 1.))]
            w = wp
        y = F.conv2d(x, w, None, stride, w.shape[-1] // 2)
        y = (y - m.view(1, -1, 1, 1)) / torch.sqrt(v.view(1, -1, 1, 1) + 1e-5) * g.view(1, -1, 1, 1) + b.view(1, -1, 1, 1)
        if residual is not None:
            y = y + residual
        return F.relu(y) if relu else y


def backbone(sd, img, arch, padded=False, engine_order=False):
    """the four stage-4 outputs of HRNet(arch) (hrnet.py:482-516), NCHW, unpadded channels"""
    arch = ARCHS[arch] if isinstance(arch, str) else arch
    P = _Params(sd, padded)
    x = P.conv_bn(img, "conv1", "bn1", 2, relu=True)
    x = P.conv_bn(x, "conv2", "bn2", 2, relu=True)
    s1 = arch.stages[0]
    for b in range(s1.num_blocks[0]):
        p = "layer1.%d." % b
        idt = P.conv_bn(x, p + "downsample.0", p + "downsample.1", 1) if p + "downsample.0.weight" in {k[9:] for k in sd} else x
        if s1.block == 'BOTTLENECK':
            o = P.conv_bn(x, p + "conv1", p + "bn1", 1, relu=True)
            o = P.conv_bn(o, p + "conv2", p + "bn2", 1, relu=True)
            x = P.conv_bn(o, p + "conv3", p + "bn3", 1, relu=True, residual=idt)
        else:
            o = P.conv_bn(x, p + "conv1", p + "bn1", 1, relu=True)
            x = P.conv_bn(o, p + "conv2", p + "bn2", 1, relu=True, residual=idt)
    xs, pre = [x], s1.widths
    for s in range(1, 4):
        st = arch.stages[s]
        new = []
        for i, t in enumerate(transition_convs(pre, st.widths)):
            if t is None:
                new.append(xs[i])
                continue
            y = xs[-1]                                                   # hrnet.py:503: the last branch of the previous stage
            for ck, bk, _, _, stride in t:
                y = P.conv_bn(y, "transition%d.%s" % (s, ck), "transition%d.%s" % (s, bk), stride, relu=True)
            new.append(y)
        xs = new
        for m in range(st.num_modules):
            p = "stage%d.%d." % (s + 1, m)
            for br, nblk in enumerate(st.num_blocks):
                for k in range(nblk):
                    q = p + "branches.%d.%d." % (br, k)
                    o = P.conv_bn(xs[br], q + "conv1", q + "bn1", 1, relu=True)
                    xs[br] = P.conv_bn(o, q + "conv2", q + "bn2", 1, relu=True, residual=xs[br])
            fuse = fuse_convs(st.widths)

            def term(i, j):
                path = fuse[i][j]
                if j > i:
                    ck, bk = path[0][:2]
                    y = P.conv_bn(xs[j], p + "fuse_layers." + ck, p + "fuse_layers." + bk, 1)
                    return F.interpolate(y, scale_factor=2 ** (j - i), mode='nearest')
                y = xs[j]
                for n, (ck, bk, *_r) in enumerate(path):
                    y = P.conv_bn(y, p + "fuse_layers." + ck, p + "fuse_layers." + bk, 2, relu=n < len(path) - 1)
                return y
            nb = len(xs)
            order = [[i] + list(range(i)) + list(range(i + 1, nb)) if engine_order else list(range(nb)) for i in range(nb)]
            out = []
            for i in range(nb):
                y = 0
                for j in order[i]:
                    y = y + (xs[j] if j == i else term(i, j))
                out.append(F.relu(y))
            xs = out
        pre = st.widths
    return [x[:, :c] for x, c in zip(xs, arch.out_widths)]


def hrfpn(sd, xs, pooling_type='AVG', engine_order=False):
    """HRFPN(stride 2, 5 outputs) (hrfpn.py:78-100) on the stage-4 outputs: the five levels, NCHW"""
    w, b = sd["neck.reduction_conv.conv.weight"], sd["neck.reduction_conv.conv.bias"]
    if engine_order:
        out, c0 = None, 0
        for i, x in enumerate(xs):
            y = F.conv2d(x, w[:, c0:c0 + x.shape[1]], b if i == 0 else None)
            c0 += x.shape[1]
            y = y if i == 0 else F.interpolate(y, scale_factor=2 ** i, mode='bilinear')
            out = y if out is None else out + y
    else:
        cat = torch.cat([xs[0]] + [F.interpolate(x, scale_factor=2 ** i, mode='bilinear') for i, x in enumerate(xs) if i > 0], 1)
        out = F.conv2d(cat, w, b)
    pool = F.max_pool2d if pooling_type == 'MAX' else F.avg_pool2d
    levels = [out] + [pool(out, kernel_size=2 ** i, stride=2 ** i) for i in range(1, 5)]
    return [F.conv2d(x, sd["neck.fpn_convs.%d.conv.weight" % i], sd["neck.fpn_convs.%d.conv.bias" % i], 2, 1)
            for i, x in enumerate(levels)]


def forward_dense(sd, img, arch, pooling_type='AVG'):
    """per level (cls_out, pts_init, pts_refine) in NCHW, and the HRFPN levels"""
    feats = hrfpn(sd, backbone(sd, img, arch), pooling_type)
    return [tr.head_single(sd, f)[:3] for f in feats], feats


def pool_cases():
    """the distinct (N, map H = W) of HRFPN's reduce / pool launches at BATCHES"""
    return sorted({(n, t // 4) for n, t in BATCHES})


def fuse_launches(arch):
    """the distinct orp_hr_fuse launches of one HRModule stage per output branch at a 1024 tile: (C padded, map side at 1024,
    number of upsampled sources)"""
    arch = ARCHS[arch] if isinstance(arch, str) else arch
    out = set()
    for st in arch.stages[1:]:
        nb = st.num_branches
        for i in range(nb - 1):
            out.add((pad8(st.widths[i]), 256 >> i, nb - 1 - i))
    return sorted(out)
