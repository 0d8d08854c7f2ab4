"""ctypes binding of liborp_b200.so (include/orp_b200.h, orp_b200_dcnv2.h, orp_b200_swin.h, orp_b200_group.h,
orp_b200_hrnet.h, orp_b200_attention.h, orp_b200_context.h, orp_b200_carafe.h).

There is NO fallback: if the shared library is missing or a call fails, an exception is raised.
The library is built in-tree by `python -m orientedreppoints_b200.build` (nvcc, sm_90a).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "liborp_b200.so")

ORP_NMS_EXACT64, ORP_NMS_COMPAT32 = 0, 1
ORP_UNION_NAN_KEEPS, ORP_UNION_GUARD, ORP_UNION_NAN_SUPPRESSES, ORP_UNION_NAN_SUPPRESSES_ALL = 0, 1, 2, 3
ORP_ORDER_INDEX_ASC, ORP_ORDER_SCORE_DESC = 0, 1
ORP_MERGE_BAD_COUNT, ORP_MERGE_BAD_TILE, ORP_MERGE_ROWS_OVERFLOW = 1, 2, 4

_vp = ctypes.c_void_p
_i = ctypes.c_int
_f = ctypes.c_float
_d = ctypes.c_double


class NmsStats(ctypes.Structure):
    _fields_ = [("pairs_total", ctypes.c_int64), ("pairs_aabb", ctypes.c_int64),
                ("pairs_clipped", ctypes.c_int64), ("pairs_fp64", ctypes.c_int64),
                ("edges", ctypes.c_int64), ("suppressing", ctypes.c_int64), ("overflow", ctypes.c_int32),
                ("rounds", ctypes.c_int32), ("n", ctypes.c_int32)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class RnmsPlan(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in ("lazy", "R", "seg_limit", "sweep_bits", "no_sync", "flags_out", "union_mode",
                                              "order", "n")] + \
              [("cap_first", ctypes.c_int64), ("cap_final", ctypes.c_int64), ("attempts", ctypes.c_int32)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class TcProblem(ctypes.Structure):
    _fields_ = [("x", _vp), ("N", _i), ("H", _i), ("W", _i), ("out", _vp), ("residual_bf16", _vp),
                ("residual_f32", _vp), ("offset", _vp), ("gn_stats", _vp), ("mask", _vp)]


class TcPlan(ctypes.Structure):
    _fields_ = [(k, _i) for k in ("BN", "stages", "grid", "num_tiles", "n_tiles_n", "ksplit", "nprob", "Cout", "Cout_padded",
                                  "split", "deform", "out_f32", "stem", "relu", "bias", "residual", "tma_epi", "ncat", "dcat",
                                  "res_mma", "b_resident", "epi_merge", "epi_bufs", "gn_fused")] + \
              [(k, _i * 5) for k in ("BW", "BH", "BI")] + [("n_pair", _i)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        for k in ("BW", "BH", "BI"):
            d[k] = list(d[k])[:self.nprob]
        return d


class GnProblem(ctypes.Structure):
    _fields_ = [("x", _vp), ("N", _i), ("H", _i), ("W", _i), ("stats", _vp), ("up_src", _vp), ("y", _vp)]


# name -> (restype, argtypes); every symbol include/orp_b200.h declares
SIGNATURES = {
    "orp_last_error": (ctypes.c_char_p, []),
    "orp_version": (_i, []),
    "orp_compiled_sm": (_i, []),
    "orp_launch_count": (ctypes.c_int64, []),
    "orp_reset_launch_count": (None, []),
    "orp_rnms": (_i, [_vp, _vp, _i, _d, _i, _i, _i, _vp, _vp, _vp]),
    "orp_poly_nms_host": (_i, [_vp, _vp, _vp, _i, _i, _f, _i]),
    "orp_rnms_last_stats": (_i, [ctypes.POINTER(NmsStats)]),
    "orp_rnms_last_plan": (_i, [ctypes.POINTER(RnmsPlan)]),
    "orp_set_timing": (None, [_i]),
    "orp_rnms_last_sweep_ms": (_i, [ctypes.POINTER(ctypes.c_float)]),
    "orp_tc_timing_collect": (_i, [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(_i), ctypes.POINTER(_d)]),
    "orp_tc_last_plan": (_i, [ctypes.POINTER(TcPlan)]),
    "orp_poly_overlaps_host": (_i, [_vp, _vp, _vp, _i, _i, _i]),
    "orp_poly_overlaps": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "orp_quad_iou_matrix": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp]),
    "orp_iou_poly_f64_pairs": (_i, [_vp, _vp, _i, _vp, _vp]),
    "orp_box_iou_rotated": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "orp_minarearect": (_i, [_vp, _i, _vp, _vp, _f, _vp, _vp]),
    "orp_head_postprocess": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _f, _d, _i, _vp, _vp, _vp, _vp, _vp]),
    "orp_head_postprocess_aug": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _f, _d, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "orp_pack_detections": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp]),
    "orp_dcn_offsets_multi": (_i, [_i, _vp, _vp, _vp, _f, _vp, _vp]),
    "orp_conv2d_f32": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _i, _vp]),
    "orp_deform_conv2d_f32": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp]),
    "orp_gn_apply_f32": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp, _f, _i, _vp, _vp, _vp]),
    "orp_maxpool3x3s2_f32": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_conv2d_bf16": (_i, [_i, ctypes.POINTER(TcProblem), _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "orp_conv2d_f16x3": (_i, [_i, ctypes.POINTER(TcProblem), _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _vp]),
    "orp_conv2d_tc_splitk": (_i, [ctypes.POINTER(TcProblem), _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_tc_plan_conv": (_i, [_i, ctypes.POINTER(TcProblem), _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i,
                              ctypes.POINTER(TcPlan)]),
    "orp_f16x3_overflow_count": (_i, [ctypes.POINTER(ctypes.c_uint), _i, _vp]),
    "orp_stem_s2d_u8_f16x3": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "orp_stem_s2d_f16x3": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "orp_stem_conv_s2d_f16x3": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _i, _vp, _vp]),
    "orp_maxpool3x3s2_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_gn_stats_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_gn_apply_f16x3_multi": (_i, [_i, _vp, _i, _i, _vp, _vp, _f, _i, _vp]),
    "orp_split_from_f32": (_i, [_vp, ctypes.c_longlong, _i, _vp, _vp]),
    "orp_split_to_f32": (_i, [_vp, ctypes.c_longlong, _i, _vp, _vp]),
    "orp_transpose_f32": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "orp_nchw_f32_to_split": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "orp_layernorm_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _f, _i, _i, _vp, _vp]),
    "orp_window_attention_bf16": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _f, _vp, _vp]),
    "orp_patch_embed_rows_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "orp_patch_embed_rows_u8_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "orp_patch_merge_gather_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_subsample2_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_layernorm_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _f, _i, _i, _vp, _vp]),
    "orp_window_attention_f16x3": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _f, _vp, _vp]),
    "orp_patch_embed_rows_f16x3": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "orp_patch_embed_rows_u8_f16x3": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "orp_patch_merge_gather_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_subsample2_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_stem_im2col_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "orp_stem_s2d_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "orp_convex_iou": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "orp_convex_giou": (_i, [_vp, _vp, _i, _vp, _vp]),
    "orp_dota_eval_task1": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _d, _i, _vp, _vp, _vp, _vp, _vp,
                                 _vp, _vp, _vp]),
    "orp_dota_eval_aoe": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _d, _vp, _vp, _vp, _vp, _vp, _vp]),
    "orp_poly2rbox_v3": (_i, [_vp, _i, _vp, _vp]),
    "orp_result_merge": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _d, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                              _vp]),
    "orp_split_tiles_u8": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _vp]),
    "orp_resize_u8": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "orp_stem_s2d_u8_padded_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "orp_stem_s2d_u8_padded_f16x3": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "orp_patch_embed_rows_u8_padded_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "orp_patch_embed_rows_u8_padded_f16x3": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "orp_stem_s2d_u8_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "orp_stem_conv_s2d_bf16": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "orp_maxpool3x3s2_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_gn_stats_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_gn_apply_bf16_multi": (_i, [_i, _vp, _i, _i, _vp, _vp, _f, _i, _vp]),
}

# name -> (restype, argtypes); every symbol include/orp_b200_dcnv2.h declares
DCNV2_SIGNATURES = {
    "orp_dcnv2_offset_mask": (_i, [_vp, ctypes.c_longlong, _vp, _vp, _vp]),
}

# name -> (restype, argtypes); every symbol include/orp_b200_swin.h declares
SWIN_SIGNATURES = {
    "orp_window_attention12_bf16": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _f, _vp, _vp]),
    "orp_window_attention12_f16x3": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _f, _vp, _vp]),
    "orp_layernorm_wide_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _f, _i, _i, _vp, _vp]),
    "orp_layernorm_wide_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _f, _i, _i, _vp, _vp]),
}

# name -> (restype, argtypes); every symbol include/orp_b200_group.h declares
GROUP_SIGNATURES = {
    "orp_group_conv2d_bf16": (_i, [ctypes.POINTER(TcProblem), _vp, _i, _i, _i, _vp, _i, _vp]),
    "orp_group_conv2d_f16x3": (_i, [ctypes.POINTER(TcProblem), _vp, _i, _i, _i, _vp, _i, _i, _vp]),
    "orp_group_conv2d_f32": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _vp]),
    "orp_tc_plan_group_conv": (_i, [_i, ctypes.POINTER(TcProblem), _vp, _i, _i, _i, _vp, _i, _i, _i, _i, ctypes.POINTER(TcPlan)]),
}

# name -> (restype, argtypes); every symbol include/orp_b200_hrnet.h declares (the pointer arrays are host arrays of device
# pointers: ctypes (c_void_p * n))
HRNET_SIGNATURES = {
    "orp_hr_fuse_bf16": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "orp_hr_fuse_f16x3": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "orp_hr_fuse_f32": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "orp_hrfpn_reduce_bf16": (_i, [_i, _vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_hrfpn_reduce_f16x3": (_i, [_i, _vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_hrfpn_reduce_f32": (_i, [_i, _vp, _i, _i, _i, _i, _vp, _vp]),
    "orp_hrfpn_pool_bf16": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "orp_hrfpn_pool_f16x3": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "orp_hrfpn_pool_f32": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
}



class GenAttentionArgs(ctypes.Structure):
    _fields_ = [(k, _vp) for k in ("q_c", "q_p", "k", "v", "pos_x", "pos_y", "out")] + \
              [(k, _i) for k in ("N", "H", "W", "Hk", "Wk", "kv_stride", "C", "heads", "ld_q", "ld_kv")]


class GenAttentionPlan(ctypes.Structure):
    _fields_ = [(k, _i) for k in ("head_dim", "queries_per_cta", "threads", "grid_x", "grid_y", "grid_z", "smem_bytes", "rx", "ry",
                                  "content", "position")]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


# name -> (restype, argtypes); every symbol include/orp_b200_attention.h declares
ATTENTION_SIGNATURES = {
    "orp_gen_attention_bf16": (_i, [ctypes.POINTER(GenAttentionArgs), _vp]),
    "orp_gen_attention_f16x3": (_i, [ctypes.POINTER(GenAttentionArgs), _vp]),
    "orp_gen_attention_f32": (_i, [ctypes.POINTER(GenAttentionArgs), _vp]),
    "orp_gen_attention_make_plan": (_i, [ctypes.POINTER(GenAttentionArgs), _i, ctypes.POINTER(GenAttentionPlan)]),
    "orp_gen_attention_bcast_add_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "orp_gen_attention_bcast_add_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "orp_gen_attention_bcast_add_f32": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp]),
}


class ContextPlan(ctypes.Structure):
    _fields_ = [(k, _i) for k in ("threads", "slots", "warps_per_slot", "chunks", "pixels_per_chunk", "grid_x", "grid_y")] + \
              [("workspace_bytes", ctypes.c_longlong)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class ContextMlp(ctypes.Structure):
    _fields_ = [(k, _vp) for k in ("w1", "b1", "ln_w", "ln_b", "w2", "b2")]


# name -> (restype, argtypes); every symbol include/orp_b200_context.h declares
CONTEXT_SIGNATURES = {
    "orp_context_make_plan": (_i, [_i, _i, _i, _i, _i, ctypes.POINTER(ContextPlan)]),
    "orp_context_pool_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, ctypes.c_size_t, _vp]),
    "orp_context_pool_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, ctypes.c_size_t, _vp]),
    "orp_context_pool_f32": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, ctypes.c_size_t, _vp]),
    "orp_context_transform": (_i, [_vp, _i, _i, _i, _i, ctypes.POINTER(ContextMlp), ctypes.POINTER(ContextMlp), _vp, _vp, _vp]),
    "orp_context_fuse_bf16": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "orp_context_fuse_f16x3": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "orp_context_fuse_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
}

# name -> (restype, argtypes); every symbol include/orp_b200_carafe.h declares
CARAFE_SIGNATURES = {
    "orp_carafe_add_bf16": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp]),
    "orp_carafe_add_f16x3": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp]),
    "orp_carafe_add_f32": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp]),
}

_LIB = None


class OrpError(RuntimeError):
    pass


def lib():
    """Load the CUDA library; raises (never falls back) when it is absent."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise OrpError(
                "liborp_b200.so not found at %s - build it with `python -m orientedreppoints_b200.build` "
                "(there is no CPU or PyTorch fallback for this path)" % LIB_PATH)
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in list(SIGNATURES.items()) + list(DCNV2_SIGNATURES.items()) + list(SWIN_SIGNATURES.items()) + \
                list(GROUP_SIGNATURES.items()) + list(HRNET_SIGNATURES.items()) + list(ATTENTION_SIGNATURES.items()) + \
                list(CONTEXT_SIGNATURES.items()) + list(CARAFE_SIGNATURES.items()):
            fn = getattr(l, name)   # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _LIB = l
    return _LIB


def check(rc, what=""):
    if rc != 0:
        msg = lib().orp_last_error()
        raise OrpError("%s failed (%d): %s" % (what, rc, msg.decode() if msg else ""))


def launch_count():
    return int(lib().orp_launch_count())


def reset_launch_count():
    lib().orp_reset_launch_count()


def last_nms_stats():
    s = NmsStats()
    check(lib().orp_rnms_last_stats(ctypes.byref(s)), "orp_rnms_last_stats")
    return s.as_dict()


def rnms_last_plan():
    """plan of this thread's most recent rotated NMS (dict of the orp_rnms_plan fields)"""
    p = RnmsPlan()
    check(lib().orp_rnms_last_plan(ctypes.byref(p)), "orp_rnms_last_plan")
    return p.as_dict()


def set_timing(on):
    lib().orp_set_timing(1 if on else 0)


def last_sweep_ms():
    v = ctypes.c_float(0)
    check(lib().orp_rnms_last_sweep_ms(ctypes.byref(v)), "orp_rnms_last_sweep_ms")
    return float(v.value)


def tc_timing_collect():
    ms, n, fl = ctypes.c_float(0), ctypes.c_int(0), ctypes.c_double(0)
    check(lib().orp_tc_timing_collect(ctypes.byref(ms), ctypes.byref(n), ctypes.byref(fl)), "orp_tc_timing_collect")
    return float(ms.value), int(n.value), float(fl.value)


def tc_last_plan():
    """launch plan of this thread's most recent tensor-core convolution (dict of the orp_tc_plan fields)"""
    p = TcPlan()
    check(lib().orp_tc_last_plan(ctypes.byref(p)), "orp_tc_last_plan")
    return p.as_dict()


def tc_plan_for(problems, cout, cout_p, kh, kw, cin, stride, pad, *, bias=False, relu=0, out_f32=False, deform=False,
                split=False, residual=0, gn=False, stem=0, ksplit=1, sms=132):
    """the plan orp_tc_plan_conv reports for a launch over problems [(N, H, W), ...] (dict of the orp_tc_plan fields); the
    pointers it passes are placeholders that the dry run only tests for NULL, so no device is needed.  residual: 0 none,
    1 16-bit, 2 fp32; gn: GroupNorm statistics requested; stem = 2: problems hold the image; ksplit > 1: the inner launch of
    the split-K convolution"""
    ph = 256                                                # a non-NULL placeholder address
    arr = (TcProblem * len(problems))()
    for q, (n, h, w) in zip(arr, problems):
        q.x, q.N, q.H, q.W, q.out = ph, n, h, w, ph
        q.residual_bf16 = ph if residual == 1 else None
        q.residual_f32 = ph if residual == 2 else None
        q.offset = ph if deform else None
        q.gn_stats = ph if gn else None
    p = TcPlan()
    check(lib().orp_tc_plan_conv(len(problems), arr, ph, cout, cout_p, kh, kw, cin, stride, pad, ph if bias else None, 0,
                                 int(relu), int(out_f32), int(deform), int(split), stem, ksplit, sms, ctypes.byref(p)),
          "orp_tc_plan_conv")
    return p.as_dict()


def tc_plan_group_for(problems, width, groups, stride, *, split=False, bias=True, relu=1, out_f32=False, residual=0, gn=False,
                      sms=132):
    """the plan orp_tc_plan_group_conv reports for a grouped 3x3 launch over problems [(N, H, W), ...] (placeholder pointers,
    no device needed); residual / gn / out_f32 / several problems are there to be refused"""
    ph = 256
    arr = (TcProblem * len(problems))()
    for q, (n, h, w) in zip(arr, problems):
        q.x, q.N, q.H, q.W, q.out = ph, n, h, w, ph
        q.residual_bf16 = ph if residual == 1 else None
        q.residual_f32 = ph if residual == 2 else None
        q.gn_stats = ph if gn else None
    p = TcPlan()
    check(lib().orp_tc_plan_group_conv(len(problems), arr, ph, width, groups, stride, ph if bias else None, int(relu), int(out_f32),
                                       int(split), sms, ctypes.byref(p)), "orp_tc_plan_group_conv")
    return p.as_dict()


GEN_ATTENTION_FORMATS = {"bf16": 0, "f16x3": 1, "fp32": 2}


def gen_attention_plan_for(fmt, N, H, W, C, heads, kv_stride, *, content=True, position=True, Hk=None, Wk=None, ld_q=None,
                           ld_kv=None):
    """the plan orp_gen_attention_make_plan reports for one attention launch in format fmt ('bf16' / 'f16x3' / 'fp32'), with
    placeholder pointers (never read, no device needed); Hk / Wk default to ceil(H / kv_stride), ceil(W / kv_stride)"""
    ph = 256
    a = GenAttentionArgs()
    a.q_c, a.k = (ph, ph) if content else (None, None)
    a.q_p, a.pos_x, a.pos_y = (ph, ph, ph) if position else (None, None, None)
    a.v, a.out = ph, 512
    a.N, a.H, a.W, a.C, a.heads, a.kv_stride = N, H, W, C, heads, kv_stride
    a.Hk = -(-H // kv_stride) if Hk is None else Hk
    a.Wk = -(-W // kv_stride) if Wk is None else Wk
    a.ld_q = 2 * C if ld_q is None else ld_q
    a.ld_kv = 2 * C if ld_kv is None else ld_kv
    p = GenAttentionPlan()
    check(lib().orp_gen_attention_make_plan(ctypes.byref(a), GEN_ATTENTION_FORMATS[fmt], ctypes.byref(p)), "orp_gen_attention_make_plan")
    return p.as_dict()


CONTEXT_FORMATS = {"bf16": 0, "f16x3": 1, "fp32": 2}


def context_plan_for(fmt, N, H, W, C):
    """the plan orp_context_make_plan reports for the pool launch of format fmt ('bf16' / 'f16x3' / 'fp32') on x [N, H, W, C]
    (no device needed)"""
    p = ContextPlan()
    check(lib().orp_context_make_plan(N, H, W, C, CONTEXT_FORMATS[fmt], ctypes.byref(p)), "orp_context_make_plan")
    return p.as_dict()


def ptr_array(ts):
    """host array of the device pointers of tensors ts (None -> NULL), for the pointer-array arguments"""
    return (ctypes.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def current_stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """device/host pointer of a torch tensor (None -> NULL)"""
    return ctypes.c_void_p(0 if t is None else t.data_ptr())
