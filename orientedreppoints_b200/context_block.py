"""The global context block (GCB) of ResNet / ResNeXt bottlenecks (mmdet/ops/context_block.py) on the engines of detector.py,
through include/orp_b200_context.h.

A block on x = bn3(conv3(.)) ([N, H, W, C] in the engine's format, before the residual add) and the block's identity runs as
  1. the pool (orp_context_pool_*): per image, the softmax over all H * W pixels of conv_mask(x) ('att') or the mean ('avg'),
     as fp32 per-chunk partials in a workspace;
  2. the transform (orp_context_transform): the partials combined, then channel_add_conv and / or sigmoid(channel_mul_conv)
     into fp32 [N, C] rows;
  3. the fuse (orp_context_fuse_*): y = relu(x * mul + add + identity).
The pool runs per image over the whole map the engine runs, padding included: a batch of tiles padded to one shape pools each
tile's padded map, the rule the GroupNorm statistics of the neck and head follow.  conv_mask's bias cancels in the softmax and
is not used.  The workspace and rows come from PyTorch's stream-ordered allocator per call, as the activations do, so a block
may run on several streams and host threads at once and inside CUDA-graph capture.
"""
import ctypes

import torch

from . import _lib
from .gen_attention import alloc, dims
from .weights import gcb_keys

_SUFFIX = {"fp32": "f32", "bf16": "bf16", "f16x3": "f16x3"}


def check_block(sd, prefix, spec):
    """ValueError unless the state dict holds exactly the context_block parameters of spec (None: none at all) under prefix
    ('backbone.layerS.I'), in their shapes"""
    p = prefix + '.context_block.'
    have = {k[len(p):]: tuple(v.shape) for k, v in sd.items() if k.startswith(p)}
    if spec is None:
        if have:
            raise ValueError("%s has a context_block but the gcb layout builds none there" % prefix)
        return
    want = gcb_keys(spec)
    if have != want:
        raise ValueError("%s.context_block with pooling_type %r, fusion_types %s on %d channels (%d planes) needs %s; the state "
                         "dict has %s" % (prefix, spec['pooling_type'], list(spec['fusion_types']), spec['channels'], spec['planes'],
                                          sorted(want.items()), sorted(have.items())))


class ContextBlock:
    """the engine form of one context_block: conv_mask's weight and the fusions' MLPs as fp32 device tensors in the
    kernels' layouts (w1 [P, C], w2 [C, P])"""

    def __init__(self, sd, prefix, spec, device):
        check_block(sd, prefix, spec)
        p = prefix + '.context_block.'
        c, pl = spec['channels'], spec['planes']
        self.spec, self.c, self.planes = spec, c, pl
        f = lambda k: sd[p + k].float().reshape(-1).to(device).contiguous()          # noqa: E731
        self.mask_w = f('conv_mask.weight') if spec['pooling_type'] == 'att' else None
        self.mlps = {}
        for fu in spec['fusion_types']:
            t = [f(fu + '_conv.%s' % k) for k in ('0.weight', '0.bias', '1.weight', '1.bias', '3.weight', '3.bias')]
            m = _lib.ContextMlp(*[x.data_ptr() for x in t])
            self.mlps[fu] = (m, t)                                            # t keeps the tensors m points into alive

    def __call__(self, eng, x, identity):
        """relu(context_block(x) + identity), in the engine's format"""
        n, h, w, c = dims(eng, x)
        assert c == self.c and dims(eng, identity) == (n, h, w, c), (dims(eng, x), dims(eng, identity), self.c)
        plan = _lib.context_plan_for(eng.name, n, h, w, c)
        ws = torch.empty(plan["workspace_bytes"] // 4, dtype=torch.float32, device=x.device)
        stream = _lib.current_stream_ptr()
        lib = _lib.lib()
        fn = "orp_context_pool_" + _SUFFIX[eng.name]
        _lib.check(getattr(lib, fn)(_lib.ptr(x), n, h, w, c, _lib.ptr(self.mask_w), _lib.ptr(ws), ws.numel() * 4, stream), fn)
        rows = {fu: torch.empty((n, c), dtype=torch.float32, device=x.device) for fu in self.mlps}
        add, mul = self.mlps.get('channel_add'), self.mlps.get('channel_mul')
        _lib.check(lib.orp_context_transform(_lib.ptr(ws), n, plan["chunks"], c, self.planes,
                                             ctypes.byref(add[0]) if add else None, ctypes.byref(mul[0]) if mul else None,
                                             _lib.ptr(rows.get('channel_add')), _lib.ptr(rows.get('channel_mul')), stream),
                   "orp_context_transform")
        y = alloc(eng, n, h, w, c)
        fn = "orp_context_fuse_" + _SUFFIX[eng.name]
        _lib.check(getattr(lib, fn)(_lib.ptr(x), _lib.ptr(identity), n, h, w, c, _lib.ptr(rows.get('channel_mul')),
                                    _lib.ptr(rows.get('channel_add')), _lib.ptr(y), stream), fn)
        return y
