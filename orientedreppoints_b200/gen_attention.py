"""The generalized attention block of ResNet backbones (mmdet/ops/generalized_attention.py, spatial_range = -1, q_stride = 1) on
the engines of detector.py, through include/orp_b200_attention.h.

A block on x (the conv2 output, [N, H, W, C] in the engine's format) runs as
  1. Qc | Qp: one 1x1 convolution of x into 2C (or C) channels, with appr_bias / geom_bias as its biases, so the kernel reads
     Qc = [t0] q + [t2] appr_bias and Qp = [t1] q + [t3] geom_bias directly;
  2. K | V: one 1x1 stride-s convolution of x (the reference's AvgPool2d(1, s) is a subsampling);
  3. one attention launch (orp_gen_attention_*) with the position tables Px / Py of this map size;
  4. proj_conv with gamma folded into its weight and bias, + x as the residual, no ReLU.
attention_type '0010' alone follows the reference's shortcut (generalized_attention.py:241-249): one attention row per image and
head (the query is appr_bias), proj_conv on that row, and a broadcast add into x.
"""
import ctypes
import math

import torch

from . import _lib
from .weights import gen_attention_keys

_SUFFIX = {"fp32": "f32", "bf16": "bf16", "f16x3": "f16x3"}


def position_table(spec, fc, n, nk):
    """fp64 [n + s (nk - 1), C]: row r = appr_geom_fc(embedding((r - s (nk - 1)) * position_magnitude)) / sqrt(2), the position
    features of generalized_attention.py:152-194, 221-238 for every coordinate difference q - s k of a query axis of n and a
    key axis of nk positions"""
    s, e = spec['kv_stride'], spec['position_embedding_dim']
    diff = (torch.arange(n + s * (nk - 1), dtype=torch.float64) - s * (nk - 1)) * spec['position_magnitude']
    dim_mat = torch.tensor([1000.0], dtype=torch.float64) ** ((4.0 / e) * torch.arange(0, e / 4, dtype=torch.float64))
    a = diff[:, None] / dim_mat[None, :]
    emb = torch.cat([a.sin(), a.cos()], 1)
    return emb @ fc.double().t() / math.sqrt(2)


def check_block(sd, prefix, spec):
    """ValueError unless the state dict holds exactly the gen_attention_block parameters of spec (None: none at all) under
    prefix ('backbone.layerS.I'), in their shapes"""
    p = prefix + '.gen_attention_block.'
    have = {k[len(p):]: tuple(v.shape) for k, v in sd.items() if k.startswith(p)}
    if spec is None:
        if have:
            raise ValueError("%s has a gen_attention_block but the gen_attention layout builds none there" % prefix)
        return
    want = gen_attention_keys(spec)
    if have != want:
        raise ValueError("%s.gen_attention_block with attention_type %s, %d heads, position_embedding_dim %d needs %s; the state "
                         "dict has %s" % (prefix, ''.join('1' if b else '0' for b in spec['attention_type']), spec['num_heads'],
                                          spec['position_embedding_dim'], sorted(want.items()), sorted(have.items())))


class GenAttentionBlock:
    """the engine form of one gen_attention_block: folded convolutions, and position tables / bias rows per shape (made on the
    first call of a shape, which capture()'s warm-up runs make outside the graph)"""

    def __init__(self, sd, prefix, spec, device):
        from .detector import ConvLayer
        check_block(sd, prefix, spec)
        p = prefix + '.gen_attention_block.'
        t, c = spec['attention_type'], spec['channels']
        self.spec, self.c, self.heads, self.s, self.device = spec, c, spec['num_heads'], spec['kv_stride'], device
        f = lambda k: sd[p + k].float().cpu()
        zw, zb = torch.zeros(c, c, 1, 1), torch.zeros(c)
        self.saliency = t == (False, False, True, False)
        ws, bs = [], []
        self.qc_off = self.qp_off = None
        if (t[0] or t[2]) and not self.saliency:
            self.qc_off = 0
            ws.append(f('query_conv.weight') if t[0] else zw)
            bs.append(f('appr_bias') if t[2] else zb)
        if t[1] or t[3]:
            self.qp_off = len(ws) * c
            ws.append(f('query_conv.weight') if t[1] else zw)
            bs.append(f('geom_bias') if t[3] else zb)
        self.q = ConvLayer(torch.cat(ws), torch.cat(bs), 1, 0, device) if ws else None
        self.k_off = 0 if (t[0] or t[2]) else None
        self.v_off = c if self.k_off is not None else 0
        kv = [f('key_conv.weight')] if self.k_off is not None else []
        self.kv = ConvLayer(torch.cat(kv + [f('value_conv.weight')]), None, self.s, 0, device)
        g = f('gamma').reshape(())
        self.proj = ConvLayer(f('proj_conv.weight') * g, f('proj_conv.bias') * g, 1, 0, device)
        self.appr_bias = f('appr_bias') if self.saliency else None
        self.fc = (f('appr_geom_fc_x.weight'), f('appr_geom_fc_y.weight')) if self.qp_off is not None else None
        self._tables, self._rows = {}, {}

    # ------------------------------------------------------------------ per-shape constants
    @staticmethod
    def _to_engine(eng, t):
        """fp32 [.., C] -> a [1, 1, R, C] tensor of the engine's format"""
        t = t.float().reshape(1, 1, -1, t.shape[-1])
        if eng.name == "fp32":
            return t.to(eng.device).contiguous()
        return eng.from_float(t)

    def tables(self, eng, h, w):
        key = (eng.name, h, w)
        if key not in self._tables:
            hk, wk = -(-h // self.s), -(-w // self.s)
            self._tables[key] = (self._to_engine(eng, position_table(self.spec, self.fc[0], w, wk)),
                                 self._to_engine(eng, position_table(self.spec, self.fc[1], h, hk)))
        return self._tables[key]

    def bias_rows(self, eng, n):
        """the '0010' shortcut's queries: appr_bias for each of n images, [n, 1, 1, C] in the engine's format"""
        key = (eng.name, n)
        if key not in self._rows:
            self._rows[key] = self._to_engine(eng, self.appr_bias.reshape(1, -1).expand(n, -1)).reshape(
                (n, 1, 1) + ((2, self.c) if eng.name == "f16x3" else (self.c,)))
        return self._rows[key]

    # ------------------------------------------------------------------ forward
    def __call__(self, eng, x):
        n, h, w, c = dims(eng, x)
        assert c == self.c, (c, self.c)
        kv = eng.conv(x, self.kv)
        hk, wk = dims(eng, kv)[1:3]
        if self.saliency:
            row = attend(eng, self.bias_rows(eng, n), 0, None, kv, self.k_off, self.v_off, None, n, 1, 1, hk, wk, self.s, c,
                         self.heads)
            y = eng.conv(row, self.proj, out_f32=True)                         # [n, 1, 1, C] fp32: gamma * proj_conv(row)
            return bcast_add(eng, x, y)
        q = eng.conv(x, self.q) if self.q is not None else None
        att = attend(eng, q, self.qc_off, self.qp_off, kv, self.k_off, self.v_off,
                     self.tables(eng, h, w) if self.qp_off is not None else None, n, h, w, hk, wk, self.s, c, self.heads)
        return eng.conv(att, self.proj, residual=x)


def dims(eng, x):
    return tuple(x.shape) if eng.name == "fp32" else eng.dims(x)


def alloc(eng, n, h, w, c):
    if eng.name == "fp32":
        return torch.empty((n, h, w, c), dtype=torch.float32, device=eng.device)
    return eng.alloc(n, h, w, c)


def _at(t, off):
    """device address of channel `off` of token 0 of t (None: NULL)"""
    return None if t is None or off is None else t.data_ptr() + off * t.element_size()


def attend(eng, q, qc_off, qp_off, kv, k_off, v_off, tables, n, h, w, hk, wk, s, c, heads):
    """one orp_gen_attention_* launch: out [n, h, w, c] in the engine's format"""
    out = alloc(eng, n, h, w, c)
    a = _lib.GenAttentionArgs()
    a.q_c, a.q_p = _at(q, qc_off), _at(q, qp_off)
    a.k, a.v = _at(kv, k_off), _at(kv, v_off)
    a.pos_x, a.pos_y = (tables[0].data_ptr(), tables[1].data_ptr()) if tables is not None else (None, None)
    a.out = out.data_ptr()
    a.N, a.H, a.W, a.Hk, a.Wk, a.kv_stride, a.C, a.heads = n, h, w, hk, wk, s, c, heads
    a.ld_q = dims(eng, q)[3] if q is not None else c
    a.ld_kv = dims(eng, kv)[3]
    fn = "orp_gen_attention_" + _SUFFIX[eng.name]
    _lib.check(getattr(_lib.lib(), fn)(ctypes.byref(a), _lib.current_stream_ptr()), fn)
    return out


def bcast_add(eng, x, row):
    """x + row[n] broadcast over the map: orp_gen_attention_bcast_add_*"""
    n, h, w, c = dims(eng, x)
    y = alloc(eng, n, h, w, c)
    fn = "orp_gen_attention_bcast_add_" + _SUFFIX[eng.name]
    _lib.check(getattr(_lib.lib(), fn)(_lib.ptr(x), n, h, w, c, _lib.ptr(row), _lib.ptr(y), _lib.current_stream_ptr()), fn)
    return y
