"""The launch plans of the wgmma convolution kernel (csrc/dense_tc.cu) that the detector uses, one parity case per plan
signature: shared by tests/test_conv_plans_gpu.py, which launches every case against fp64, and tests/test_tc_plan_cpu.py,
which plans every case through the dry run (orp_tc_plan_conv) without a device."""
from types import SimpleNamespace

SIG_FIELDS = ("precision", "deform", "out", "BN", "tma_epi", "ncat", "dcat", "residual", "b_resident", "epi_merge", "epi_bufs",
              "gn_fused", "stages", "relu", "bias", "ksplit>1", "nprob>1", "tiles>grid", "Cout%BN", "stem")


def signature(p):
    """the plan reduced to what selects kernel code paths (residual: 0 none, 1 16-bit, 2 fp32; stem: 2 space-to-depth conv1)"""
    return ("f16x3" if p["split"] else "bf16", p["deform"], "f32" if p["out_f32"] else ("split" if p["split"] else "bf16"),
            p["BN"], p["tma_epi"], p["ncat"], p["dcat"], p["residual"], p["b_resident"], p["epi_merge"], p["epi_bufs"],
            p["gn_fused"], p["stages"], p["relu"], p["bias"], int(p["ksplit"] > 1), int(p["nprob"] > 1),
            int(p["num_tiles"] > p["grid"]), int(p["Cout"] % p["BN"] != 0), p["stem"])


# One case per production plan signature: (signature, precision, kind, Cin, Cout, k, stride, bias, act, out_f32, residual,
# gn, problems).  kind "conv": a k x k convolution (pad k // 2) of every problem (N, H, W), launched the way the engine
# launches it (split-K where EngineTC._ksplit picks it); "deform": the head's DCN over the problems; "stem": conv1 in
# space-to-depth form over N images of H x W.  act: 1 ReLU, 2 exact GELU; residual: 1 16-bit, 2 fp32.  The comment above
# a case names the production layers (workload, layer) that launch its plan.  Shapes are the smallest that reach the
# plan with output maps that are not multiples of the tile box (or image counts not multiples of BI) and, where production
# runs several tiles per CTA, more than two tiles per CTA.
PARITY = [
    # r101 stem, r50 stem
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 1, 1, 0, 0, 1, 0, 2), 'f16x3', 'stem', 64, 64, 4, 1, 1, 1, 0, 0, 0, [(5, 106, 130)]),
    # r101 ds0, r50 ds0
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 1, 1, 2, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 64, 256, 1, 1, 1, 0, 0, 0, 0, [(1, 133, 130)]),
    # r101 c1_0, r50 c1_0
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 1, 1, 2, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 64, 64, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r101 c2_0, r50 c2_0
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 64, 64, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r101 c3_0, r50 c3_0
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 1, 1, 2, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 64, 256, 1, 1, 1, 1, 0, 1, 0, [(1, 133, 130)]),
    # r101 c1_0, r50 c1_0
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 64, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r101 ds1, r101 ds2, r50 ds1, r50 ds2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 512, 1, 2, 1, 0, 0, 0, 0, [(2, 133, 130)]),
    # r101 c1_1, r50 c1_1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 1, 1, 0, 2, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 128, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r101 c2_1, r50 c2_1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 0, 2, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 128, 128, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r101 c3_1, r101 c3_2, r101 c3_3, r50 c3_1, r50 c3_2, r50 c3_3
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 0, 1, 1, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 128, 512, 1, 1, 1, 1, 0, 1, 0, [(2, 67, 67)]),
    # r101 c1_2, r50 c1_2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 512, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r101 c1_3, r50 c1_2, r50 c1_3, r50 c2_2, r50 c2_3
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 1024, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r101 ds3, r50 ds3, swin qkv3
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 768, 2304, 1, 1, 1, 0, 0, 0, 0, [(4, 25, 17)]),
    # r101 lat, r50 lat, swin lat
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 1, 3, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 192, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 133, 130)]),
    # r101 fpn, r50 fpn, r50 lat, swin fpn
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 1, 3, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 1024, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 133, 130)]),
    # r101 fpn, r101 lat, r50 fpn, r50 lat
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 1, 3, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 1024, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 130, 118)]),
    # r101 fpn, r101 lat, r50 fpn, r50 lat, r50 p6
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 0, 1, 1, 3, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 1024, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 4, 8)]),
    # r101 p6, r50 fpn, r50 p7
    (('f16x3', 0, 'f32', 128, 0, 0, 0, 0, 0, 0, 1, 0, 5, 0, 0, 1, 0, 1, 0, 0), 'f16x3', 'conv', 256, 256, 3, 1, 0, 0, 0, 0, 1, [(4, 11, 18)]),
    # r101 tower, r50 tower, swin tower
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 1, 3, 0, 0, 0, 1, 1, 0, 0), 'f16x3', 'conv', 256, 256, 3, 1, 0, 0, 0, 0, 1, [(2, 115, 79), (2, 58, 40), (2, 29, 20), (2, 15, 10), (2, 8, 5)]),
    # r101 init_conv, r50 init_conv, swin init_conv
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 1, 1, 0, 0), 'f16x3', 'conv', 256, 256, 3, 1, 1, 1, 0, 0, 0, [(2, 97, 67), (2, 49, 34), (2, 25, 17), (2, 13, 9), (2, 7, 5)]),
    # r101 cls_out, r101 init_out, r50 cls_out, r50 init_out, swin cls_out, swin init_out
    (('f16x3', 0, 'f32', 32, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 1, 1, 1, 0), 'f16x3', 'conv', 256, 15, 1, 1, 1, 0, 1, 0, 0, [(2, 97, 67), (2, 49, 34), (2, 25, 17), (2, 13, 9), (2, 7, 5)]),
    # r101 dcn, r50 dcn, swin dcn
    (('f16x3', 1, 'split', 128, 1, 0, 1, 0, 0, 0, 1, 0, 2, 1, 0, 0, 1, 1, 0, 0), 'f16x3', 'deform', 256, 256, 3, 1, 0, 1, 0, 0, 0, [(5, 33, 33), (5, 17, 17), (5, 9, 9), (5, 5, 5), (5, 3, 3)]),
    # r101 ref_out, r50 ref_out, swin ref_out
    (('f16x3', 0, 'f32', 32, 0, 0, 0, 2, 1, 0, 2, 0, 6, 0, 1, 0, 1, 1, 1, 0), 'f16x3', 'conv', 256, 18, 1, 1, 1, 0, 1, 2, 0, [(2, 97, 67), (2, 49, 34), (2, 25, 17), (2, 13, 9), (2, 7, 5)]),
    # r101 c1_3, r101 c2_3, r50 c1_3, r50 c2_1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 0, 2, 1, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 1024, 512, 1, 1, 1, 1, 0, 0, 0, [(3, 40, 31)]),
    # r50 c1_1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 1, 1, 0, 2, 1, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 512, 128, 1, 1, 1, 1, 0, 0, 0, [(1, 130, 118)]),
    # r50 ds2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 0, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 512, 1024, 1, 2, 1, 0, 0, 0, 0, [(3, 79, 61)]),
    # r50 c1_2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 1, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 512, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 130, 118)]),
    # r50 c1_2, r50 c1_3, r50 c2_2
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 1024, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 4, 4)]),
    # r50 c3_2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 0, 1, 1, 0, 3, 1, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 256, 1024, 1, 1, 1, 1, 0, 1, 0, [(3, 40, 31)]),
    # r50 ds3
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 0, 2, 0, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 1024, 2048, 1, 2, 1, 0, 0, 0, 0, [(4, 29, 29)]),
    # r50 c2_3
    (('f16x3', 0, 'f32', 256, 0, 0, 0, 0, 0, 0, 1, 0, 3, 0, 0, 1, 0, 1, 0, 0), 'f16x3', 'conv', 512, 512, 3, 1, 1, 1, 0, 0, 0, [(4, 11, 18)]),
    # r50 c3_3
    (('f16x3', 0, 'split', 128, 1, 0, 0, 1, 0, 1, 2, 0, 3, 1, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 512, 2048, 1, 1, 1, 1, 0, 1, 0, [(1, 29, 31)]),
    # r50 lat
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 1, 3, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 512, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 130, 118)]),
    # r101 p7, r50 p6, r50 p7
    (('f16x3', 0, 'f32', 64, 0, 0, 0, 0, 0, 0, 1, 0, 6, 0, 0, 1, 0, 0, 0, 0), 'f16x3', 'conv', 256, 256, 3, 2, 0, 0, 0, 0, 1, [(1, 4, 4)]),
    # r101 c1_2, r101 c2_2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 1024, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 130, 118)]),
    # swin embed
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 1, 1, 1, 0, 3, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 64, 96, 1, 1, 1, 0, 0, 0, 0, [(1, 133, 130)]),
    # swin qkv0
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 1, 1, 1, 0, 3, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 96, 288, 1, 1, 1, 0, 0, 0, 0, [(3, 33, 33)]),
    # swin proj0
    (('f16x3', 0, 'split', 128, 1, 0, 0, 1, 1, 1, 2, 0, 3, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 96, 96, 1, 1, 1, 0, 0, 1, 0, [(1, 133, 130)]),
    # swin fc1_0
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 1, 1, 0, 2, 2, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 96, 384, 1, 1, 1, 2, 0, 0, 0, [(5, 33, 33)]),
    # swin fc2_0
    (('f16x3', 0, 'split', 128, 1, 0, 0, 1, 0, 1, 2, 0, 3, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 384, 96, 1, 1, 1, 0, 0, 1, 0, [(1, 133, 130)]),
    # swin red0
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 0, 0, 0, 0, 1, 1, 0), 'f16x3', 'conv', 384, 192, 1, 1, 0, 0, 0, 0, 0, [(1, 133, 130)]),
    # swin qkv1
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 1, 1, 1, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 192, 576, 1, 1, 1, 0, 0, 0, 0, [(5, 17, 17)]),
    # swin fc2_1, swin proj1
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 0, 1, 1, 0, 3, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 192, 192, 1, 1, 1, 0, 0, 1, 0, [(1, 133, 130)]),
    # swin fc1_1, swin fc1_2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 2, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 192, 768, 1, 1, 1, 2, 0, 0, 0, [(5, 33, 33)]),
    # swin red1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 0, 2, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 768, 384, 1, 1, 0, 0, 0, 0, 0, [(5, 33, 33)]),
    # swin qkv2
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 1, 1, 0, 2, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 384, 1152, 1, 1, 1, 0, 0, 0, 0, [(4, 25, 17)]),
    # swin fc2_2, swin proj2
    (('f16x3', 0, 'split', 128, 1, 0, 0, 1, 0, 1, 2, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 384, 384, 1, 1, 1, 0, 0, 1, 0, [(5, 33, 33)]),
    # swin red2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 1536, 768, 1, 1, 0, 0, 0, 0, 0, [(5, 33, 33)]),
    # swin fc2_3, swin proj3
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 0, 1, 1, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 768, 768, 1, 1, 1, 0, 0, 1, 0, [(5, 33, 33)]),
    # swin fc1_3
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 2, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 768, 3072, 1, 1, 1, 2, 0, 0, 0, [(4, 17, 17)]),
    # swin fpn, swin lat
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 1, 2, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 768, 256, 1, 1, 0, 0, 0, 0, 1, [(2, 61, 64)]),
    # swin embed, swin qkv0
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 64, 96, 1, 1, 1, 0, 0, 0, 0, [(5, 33, 33)]),
    # swin fc2_0, swin proj0
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 1, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 96, 96, 1, 1, 1, 0, 0, 1, 0, [(5, 33, 33)]),
    # swin fc1_0
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 1, 0, 2, 0, 6, 2, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 96, 384, 1, 1, 1, 2, 0, 0, 0, [(5, 33, 33)]),
    # swin red0
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 1, 0, 2, 0, 6, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 384, 192, 1, 1, 0, 0, 0, 0, 0, [(5, 33, 33)]),
    # swin qkv1
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 192, 576, 1, 1, 1, 0, 0, 0, 0, [(5, 17, 17)]),
    # swin proj1
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 1, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 192, 192, 1, 1, 1, 0, 0, 1, 0, [(5, 33, 33)]),
    # swin fc1_1, swin fc1_2
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 0, 3, 2, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 192, 768, 1, 1, 1, 2, 0, 0, 0, [(5, 33, 33)]),
    # swin fc2_1
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 1, 0, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 768, 192, 1, 1, 1, 0, 0, 1, 0, [(5, 33, 33)]),
    # swin red1
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 0, 0, 1, 0, 5, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 768, 384, 1, 1, 0, 0, 0, 0, 0, [(5, 33, 33)]),
    # swin qkv2
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 0, 0, 2, 0, 4, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 384, 1152, 1, 1, 1, 0, 0, 0, 0, [(4, 25, 17)]),
    # swin fc2_2, swin proj2
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 1, 0, 0, 2, 0, 4, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 384, 384, 1, 1, 1, 0, 0, 1, 0, [(5, 33, 33)]),
    # swin red2
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 1536, 768, 1, 1, 0, 0, 0, 0, 0, [(5, 33, 33)]),
    # r50 ds3, swin qkv3
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 768, 2304, 1, 1, 1, 0, 0, 0, 0, [(4, 25, 17)]),
    # swin fc2_3, swin proj3
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 1, 0, 0, 2, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 768, 768, 1, 1, 1, 0, 0, 1, 0, [(5, 33, 33)]),
    # swin fc1_3
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 2, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 768, 3072, 1, 1, 1, 2, 0, 0, 0, [(4, 17, 17)]),
    # r50 lat, swin lat
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 1, 3, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 192, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 133, 130)]),
    # swin fpn, swin lat
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 0, 0, 1, 1, 5, 0, 0, 0, 0, 0, 0, 0), 'bf16', 'conv', 768, 256, 1, 1, 0, 0, 0, 0, 1, [(2, 61, 64)]),
    # r50 fpn, r50 lat, swin fpn
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 1, 3, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 1024, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 133, 130)]),
    # r50 tower, swin tower
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 1, 3, 0, 0, 0, 1, 1, 0, 0), 'bf16', 'conv', 256, 256, 3, 1, 0, 0, 0, 0, 1, [(2, 115, 79), (2, 58, 40), (2, 29, 20), (2, 15, 10), (2, 8, 5)]),
    # r50 init_conv, swin init_conv
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 1, 1, 0, 0), 'bf16', 'conv', 256, 256, 3, 1, 1, 1, 0, 0, 0, [(2, 97, 67), (2, 49, 34), (2, 25, 17), (2, 13, 9), (2, 7, 5)]),
    # r50 cls_out, r50 init_out, swin cls_out, swin init_out
    (('bf16', 0, 'f32', 32, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 1, 1, 1, 0), 'bf16', 'conv', 256, 15, 1, 1, 1, 0, 1, 0, 0, [(2, 97, 67), (2, 49, 34), (2, 25, 17), (2, 13, 9), (2, 7, 5)]),
    # r50 dcn, swin dcn
    (('bf16', 1, 'bf16', 128, 1, 0, 0, 0, 0, 0, 1, 0, 3, 1, 0, 0, 1, 1, 0, 0), 'bf16', 'deform', 256, 256, 3, 1, 0, 1, 0, 0, 0, [(5, 33, 33), (5, 17, 17), (5, 9, 9), (5, 5, 5), (5, 3, 3)]),
    # r50 ref_out, swin ref_out
    (('bf16', 0, 'f32', 32, 0, 0, 0, 2, 1, 0, 2, 0, 6, 0, 1, 0, 1, 1, 1, 0), 'bf16', 'conv', 256, 18, 1, 1, 1, 0, 1, 2, 0, [(2, 97, 67), (2, 49, 34), (2, 25, 17), (2, 13, 9), (2, 7, 5)]),
    # r50 stem
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 0, 2), 'bf16', 'stem', 64, 64, 4, 1, 1, 1, 0, 0, 0, [(5, 106, 130)]),
    # r50 ds0
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 64, 256, 1, 1, 1, 0, 0, 0, 0, [(1, 133, 130)]),
    # r50 c1_0
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 64, 64, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r50 c2_0
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 1, 0, 1, 0, 6, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 64, 64, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r50 c3_0
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 1, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 64, 256, 1, 1, 1, 1, 0, 1, 0, [(1, 133, 130)]),
    # r50 ds1, r50 ds2
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 256, 512, 1, 2, 1, 0, 0, 0, 0, [(2, 133, 130)]),
    # r50 c1_1
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 1, 0, 2, 0, 5, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 256, 128, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r50 c2_1
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 0, 0, 1, 0, 5, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 128, 128, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r50 c3_1
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 1, 1, 0, 2, 0, 5, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 128, 512, 1, 1, 1, 1, 0, 1, 0, [(2, 67, 67)]),
    # r50 c1_1
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 0, 0, 2, 0, 4, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 512, 128, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r50 c1_2
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 512, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r50 c1_2, r50 c1_3, r50 c2_2, r50 c2_3
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 1024, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 130)]),
    # r50 c3_2, r50 c3_3
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 1, 0, 0, 2, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 256, 1024, 1, 1, 1, 1, 0, 1, 0, [(5, 25, 33)]),
    # r50 fpn, r50 lat
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 1, 3, 0, 0, 0, 0, 0, 0, 0), 'bf16', 'conv', 2048, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 130, 118)]),
    # r50 p6
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 0, 0, 1, 1, 6, 0, 0, 0, 0, 0, 0, 0), 'bf16', 'conv', 2048, 256, 3, 2, 0, 0, 0, 0, 1, [(5, 37, 43)]),
    # r50 p7
    (('bf16', 0, 'f32', 128, 0, 0, 0, 0, 0, 0, 1, 0, 5, 0, 0, 1, 0, 1, 0, 0), 'bf16', 'conv', 256, 256, 3, 2, 0, 0, 0, 0, 1, [(4, 33, 23)]),
    # ---- the ResNeXt, HRNet + HRFPN, DCN-stage and GeneralizedAttention graphs (16 x 1024^2, 4 x 960^2): the layer names are
    # the reference's module paths; HRNet's widths are padded to multiples of 8 (W18: 24 / 40 / 72 / 144), so each case keeps
    # the Cin (partial 64-channel K block, or a Cin below one block) and Cout (padded up inside the BN tile) of its layers
    # hrnet-w18 bf16 x16 fpn_convs.2: Cin 256 x Cout 256 k3 s2
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 0, 1, 0, 0, 0, 0, 0), 'bf16', 'conv', 256, 256, 3, 2, 1, 0, 0, 0, 0, [(6, 81, 123)]),
    # r50-ga bf16 x16 layer4.*.att.kv: Cin 512 x Cout 1024 k1 s2
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 0, 3, 0, 0, 0, 0, 0, 0, 0), 'bf16', 'conv', 512, 1024, 1, 2, 0, 0, 0, 0, 0, [(6, 155, 15)]),
    # r50-ga bf16 x16 layer3.*.att.kv: Cin 256 x Cout 512 k1 s2
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 0, 3, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 256, 512, 1, 2, 0, 0, 0, 0, 0, [(6, 35, 139)]),
    # x101-64x4d bf16 x16 layer1.*.c1: Cin 64 x Cout 256 k1 s1
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 64, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 stage4.*.branches.3.*.conv1: Cin 144 x Cout 144 k3 s1 (the plan also runs Cin x Cout 256x24)
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 0, 0, 0, 1, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 144, 144, 3, 1, 1, 1, 0, 0, 0, [(3, 33, 33)]),
    # hrnet-w18 bf16 x16 stage3.*.branches.2.*.conv1, stage4.*.branches.2.*.conv1: Cin 72 x Cout 72 k3 s1 (the plan also runs Cin x Cout 72x144)
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 0, 1, 0, 1, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 72, 72, 3, 1, 1, 1, 0, 0, 0, [(5, 33, 33)]),
    # hrnet-w18 bf16 x16 stage4.*.fuse_layers.0.3.0: Cin 144 x Cout 24 k1 s1
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 0, 1, 0), 'bf16', 'conv', 144, 24, 1, 1, 1, 0, 0, 0, 0, [(1, 2, 2)]),
    # hrnet-w18 bf16 x16 stage2.*.fuse_layers.0.1.0, stage3.*.fuse_layers.0.1.0, stage4.*.fuse_layers.0.1.0: Cin 40 x Cout 24 k1 s1 (the plan also runs Cin x Cout 72x24, 144x72)
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 40, 24, 1, 1, 1, 0, 0, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 stage2.*.branches.0.*.conv1, stage3.*.branches.0.*.conv1, stage4.*.branches.0.*.conv1: Cin 24 x Cout 24 k3 s1 (the plan also runs Cin x Cout 40x72)
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 0, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 24, 24, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 stage4.*.branches.3.*.conv2: Cin 144 x Cout 144 k3 s1
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 1, 0, 0, 2, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 144, 144, 3, 1, 1, 1, 0, 1, 0, [(3, 33, 33)]),
    # hrnet-w18 bf16 x16 stage3.*.fuse_layers.2.0.1, stage4.*.fuse_layers.2.0.1: Cin 24 x Cout 72 k3 s2 (the plan also runs Cin x Cout 24x144, 40x72, 40x144)
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 1, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 24, 72, 3, 2, 1, 0, 0, 1, 0, [(5, 65, 65)]),
    # hrnet-w18 bf16 x16 stage2.*.branches.0.*.conv2, stage3.*.branches.0.*.conv2, stage4.*.branches.0.*.conv2: Cin 24 x Cout 24 k3 s1 (the plan also runs Cin x Cout 40x72, 72x72, 72x144)
    (('bf16', 0, 'bf16', 32, 0, 0, 0, 1, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 24, 24, 3, 1, 1, 1, 0, 1, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 transition1.1.0: Cin 256 x Cout 40 k3 s2
    (('bf16', 0, 'bf16', 64, 0, 0, 0, 0, 0, 0, 1, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 256, 40, 3, 2, 1, 1, 0, 0, 0, [(5, 105, 129)]),
    # hrnet-w18 bf16 x16 stage4.*.fuse_layers.1.3.0: Cin 144 x Cout 40 k1 s1
    (('bf16', 0, 'bf16', 64, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 0, 1, 0), 'bf16', 'conv', 144, 40, 1, 1, 1, 0, 0, 0, 0, [(1, 2, 2)]),
    # hrnet-w18 bf16 x16 stage3.*.fuse_layers.1.2.0, stage4.*.fuse_layers.1.2.0: Cin 72 x Cout 40 k1 s1
    (('bf16', 0, 'bf16', 64, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 72, 40, 1, 1, 1, 0, 0, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 stage2.*.branches.1.*.conv1, stage3.*.branches.1.*.conv1, stage4.*.branches.1.*.conv1: Cin 40 x Cout 40 k3 s1
    (('bf16', 0, 'bf16', 64, 0, 0, 0, 0, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 40, 40, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 stage3.*.fuse_layers.1.0.0, stage4.*.fuse_layers.1.0.0: Cin 24 x Cout 40 k3 s2
    (('bf16', 0, 'bf16', 64, 0, 0, 0, 1, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 24, 40, 3, 2, 1, 0, 0, 1, 0, [(5, 105, 129)]),
    # hrnet-w18 bf16 x16 stage2.*.branches.1.*.conv2, stage3.*.branches.1.*.conv2, stage4.*.branches.1.*.conv2: Cin 40 x Cout 40 k3 s1 (the plan also runs Cin x Cout 24x40)
    (('bf16', 0, 'bf16', 64, 0, 0, 0, 1, 1, 0, 2, 0, 6, 1, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 40, 40, 3, 1, 1, 1, 0, 1, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 fpn_convs.3: Cin 256 x Cout 256 k3 s2
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 0, 0, 1, 0, 6, 0, 1, 0, 0, 0, 0, 0), 'bf16', 'conv', 256, 256, 3, 2, 1, 0, 0, 0, 0, [(6, 11, 113)]),
    # hrnet-w18 bf16 x16 reduction_conv.3: Cin 144 x Cout 256 k1 s1
    (('bf16', 0, 'f32', 256, 0, 0, 0, 0, 0, 0, 2, 0, 3, 0, 0, 0, 0, 0, 0, 0), 'bf16', 'conv', 144, 256, 1, 1, 0, 0, 1, 0, 0, [(1, 120, 127)]),
    # hrnet-w18 bf16 x16 reduction_conv.1: Cin 40 x Cout 256 k1 s1 (the plan also runs Cin x Cout 72x256)
    (('bf16', 0, 'f32', 256, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 40, 256, 1, 1, 0, 0, 1, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 bf16 x16 reduction_conv.0: Cin 24 x Cout 256 k1 s1
    (('bf16', 0, 'f32', 256, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 24, 256, 1, 1, 1, 0, 1, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x4@960 reduction_conv.2: Cin 72 x Cout 256 k1 s1
    (('f16x3', 0, 'f32', 128, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 72, 256, 1, 1, 0, 0, 1, 0, 0, [(1, 83, 91)]),
    # hrnet-w18 f16x3 x16 reduction_conv.3: Cin 144 x Cout 256 k1 s1 (the plan also runs Cin x Cout 256x256)
    (('f16x3', 0, 'f32', 256, 0, 0, 0, 0, 0, 0, 2, 0, 3, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 144, 256, 1, 1, 0, 0, 1, 0, 0, [(1, 120, 127)]),
    # hrnet-w18 f16x3 x16 reduction_conv.2: Cin 72 x Cout 256 k1 s1 (the plan also runs Cin x Cout 128x256)
    (('f16x3', 0, 'f32', 256, 0, 0, 0, 0, 0, 0, 2, 0, 3, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 72, 256, 1, 1, 0, 0, 1, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x16/f16x3 x4@960 reduction_conv.1: Cin 40 x Cout 256 k1 s1 (the plan also runs Cin x Cout 64x256)
    (('f16x3', 0, 'f32', 256, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 40, 256, 1, 1, 0, 0, 1, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x16/f16x3 x4@960 reduction_conv.0: Cin 24 x Cout 256 k1 s1 (the plan also runs Cin x Cout 32x256)
    (('f16x3', 0, 'f32', 256, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 24, 256, 1, 1, 1, 0, 1, 0, 0, [(1, 133, 129)]),
    # r50-dcn f16x3 x16 layer4.*.off: Cin 512 x Cout 18 k3 s1 (the plan also runs Cin x Cout 512x27)
    (('f16x3', 0, 'f32', 32, 0, 0, 0, 0, 0, 0, 1, 0, 6, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 512, 18, 3, 1, 1, 0, 1, 0, 0, [(1, 2, 2)]),
    # r50-dcn f16x3 x16 layer3.*.off: Cin 256 x Cout 18 k3 s1 (the plan also runs Cin x Cout 128x18, 128x27, 256x27)
    (('f16x3', 0, 'f32', 32, 0, 0, 0, 0, 0, 0, 1, 0, 6, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 256, 18, 3, 1, 1, 0, 1, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x4@960 reduction_conv.3: Cin 144 x Cout 256 k1 s1
    (('f16x3', 0, 'f32', 64, 0, 0, 0, 0, 1, 0, 2, 0, 6, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 144, 256, 1, 1, 0, 0, 1, 0, 0, [(1, 2, 2)]),
    # hrnet-w32 f16x3 x16 stage3.*.branches.2.*.conv2, stage4.*.branches.2.*.conv2: Cin 128 x Cout 128 k3 s1 (the plan also runs Cin x Cout 64x128)
    (('f16x3', 0, 'split', 128, 1, 0, 0, 1, 0, 1, 2, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 128, 128, 3, 1, 1, 1, 0, 1, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x16 stage3.*.branches.2.*.conv2, stage4.*.branches.2.*.conv2: Cin 72 x Cout 72 k3 s1 (the plan also runs Cin x Cout 40x72)
    (('f16x3', 0, 'split', 128, 1, 0, 0, 1, 0, 1, 2, 0, 3, 1, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 72, 72, 3, 1, 1, 1, 0, 1, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x4@960 fpn_convs.1: Cin 256 x Cout 256 k3 s2
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 0, 2, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 256, 3, 2, 1, 0, 0, 0, 0, [(6, 35, 139)]),
    # hrnet-w18 f16x3 x16 stage3.*.branches.2.*.conv1, stage4.*.branches.2.*.conv1: Cin 72 x Cout 72 k3 s1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 0, 2, 1, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 72, 72, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 129)]),
    # r50-ga f16x3 x4@960 fpn1; x101-64x4d f16x3 x4@960 fpn1: Cin 256 x Cout 256 k3 s1 (the plan also runs Cin x Cout 1024x256)
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 0, 1, 1, 2, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 256, 3, 1, 0, 0, 0, 0, 1, [(1, 83, 91)]),
    # hrnet-w32 f16x3 x16 stage4.*.fuse_layers.2.3.0: Cin 256 x Cout 128 k1 s1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 1, 1, 0, 2, 0, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 256, 128, 1, 1, 1, 0, 0, 0, 0, [(1, 120, 127)]),
    # hrnet-w18 f16x3 x16 stage4.*.fuse_layers.2.3.0: Cin 144 x Cout 72 k1 s1
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 1, 1, 0, 2, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 144, 72, 1, 1, 1, 0, 0, 0, 0, [(1, 120, 127)]),
    # hrnet-w18 f16x3 x16 transition2.2.0: Cin 40 x Cout 72 k3 s2
    (('f16x3', 0, 'split', 128, 1, 1, 0, 0, 0, 1, 1, 0, 2, 1, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 40, 72, 3, 2, 1, 1, 0, 0, 0, [(5, 105, 129)]),
    # hrnet-w18 f16x3 x16 fpn_convs.2; hrnet-w32 f16x3 x16 fpn_convs.2: Cin 256 x Cout 256 k3 s2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 0, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 256, 256, 3, 2, 1, 0, 0, 0, 0, [(6, 81, 123)]),
    # hrnet-w18 f16x3 x16 stage4.*.branches.3.*.conv1: Cin 144 x Cout 144 k3 s1 (the plan also runs Cin x Cout 72x144)
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 144, 144, 3, 1, 1, 1, 0, 0, 0, [(1, 120, 127)]),
    # r50-ga f16x3 x16 layer4.*.att.kv: Cin 512 x Cout 1024 k1 s2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 512, 1024, 1, 2, 0, 0, 0, 0, 0, [(6, 155, 15)]),
    # r50-ga f16x3 x16 layer3.*.att.kv: Cin 256 x Cout 512 k1 s2
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 0, 1, 1, 0, 3, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 512, 1, 2, 0, 0, 0, 0, 0, [(6, 35, 139)]),
    # x101-64x4d f16x3 x16/f16x3 x4@960 layer1.*.c1; x50-32x8d f16x3 x16 layer1.*.c1: Cin 64 x Cout 256 k1 s1
    (('f16x3', 0, 'split', 256, 1, 0, 0, 0, 1, 1, 2, 0, 3, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 64, 256, 1, 1, 1, 1, 0, 0, 0, [(1, 133, 129)]),
    # hrnet-w32 f16x3 x16 stage4.*.fuse_layers.3.0.2: Cin 32 x Cout 256 k3 s2 (the plan also runs Cin x Cout 64x256)
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 0, 1, 1, 0, 3, 0, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 32, 256, 3, 2, 1, 0, 0, 1, 0, [(6, 81, 123)]),
    # hrnet-w18 f16x3 x16 stage4.*.fuse_layers.3.0.2: Cin 24 x Cout 144 k3 s2 (the plan also runs Cin x Cout 40x144)
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 0, 1, 1, 0, 3, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 24, 144, 3, 2, 1, 0, 0, 1, 0, [(6, 81, 123)]),
    # hrnet-w18 f16x3 x16 stage4.*.branches.3.*.conv2: Cin 144 x Cout 144 k3 s1 (the plan also runs Cin x Cout 72x144)
    (('f16x3', 0, 'split', 256, 1, 0, 0, 1, 0, 1, 1, 0, 3, 1, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 144, 144, 3, 1, 1, 1, 0, 1, 0, [(1, 120, 127)]),
    # hrnet-w18 f16x3 x4@960 stage4.*.fuse_layers.3.0.2: Cin 24 x Cout 144 k3 s2 (the plan also runs Cin x Cout 40x144)
    (('f16x3', 0, 'split', 64, 1, 0, 0, 1, 0, 1, 2, 0, 4, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 24, 144, 3, 2, 1, 0, 0, 1, 0, [(1, 2, 2)]),
    # hrnet-w32 f16x3 x16 stage3.*.fuse_layers.1.0.0, stage4.*.fuse_layers.1.0.0: Cin 32 x Cout 64 k3 s2 (the plan also runs Cin x Cout 512x512)
    (('f16x3', 0, 'split', 64, 1, 0, 0, 1, 0, 1, 2, 0, 4, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 32, 64, 3, 2, 1, 0, 0, 1, 0, [(5, 105, 129)]),
    # hrnet-w18 f16x3 x16/f16x3 x4@960 stage3.*.fuse_layers.1.0.0, stage4.*.fuse_layers.1.0.0: Cin 24 x Cout 40 k3 s2 (the plan also runs Cin x Cout 24x72, 40x72)
    (('f16x3', 0, 'split', 64, 1, 0, 0, 1, 0, 1, 2, 0, 4, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 24, 40, 3, 2, 1, 0, 0, 1, 0, [(5, 105, 129)]),
    # hrnet-w18 f16x3 x4@960 stage4.*.branches.3.*.conv2: Cin 144 x Cout 144 k3 s1 (the plan also runs Cin x Cout 72x144)
    (('f16x3', 0, 'split', 64, 1, 0, 0, 1, 0, 1, 2, 0, 4, 1, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 144, 144, 3, 1, 1, 1, 0, 1, 0, [(1, 2, 2)]),
    # hrnet-w32 f16x3 x16 stage2.*.fuse_layers.1.0.0: Cin 32 x Cout 64 k3 s2 (the plan also runs Cin x Cout 64x64)
    (('f16x3', 0, 'split', 64, 1, 0, 0, 1, 0, 1, 2, 0, 4, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 32, 64, 3, 2, 1, 1, 0, 1, 0, [(5, 105, 129)]),
    # hrnet-w18 f16x3 x16/f16x3 x4@960 stage2.*.branches.0.*.conv2, stage3.*.branches.0.*.conv2, stage4.*.branches.0.*.conv2: Cin 24 x Cout 24 k3 s1 (the plan also runs Cin x Cout 24x40, 32x32, 40x40, 40x72, 72x72)
    (('f16x3', 0, 'split', 64, 1, 0, 0, 1, 0, 1, 2, 0, 4, 1, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 24, 24, 3, 1, 1, 1, 0, 1, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x4@960 fpn_convs.2; hrnet-w18 f16x3 x16 fpn_convs.3; hrnet-w32 f16x3 x16 fpn_convs.3: Cin 256 x Cout 256 k3 s2
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 0, 1, 0, 3, 0, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 256, 256, 3, 2, 1, 0, 0, 0, 0, [(6, 11, 113)]),
    # hrnet-w18 f16x3 x4@960 stage4.*.branches.3.*.conv1: Cin 144 x Cout 144 k3 s1 (the plan also runs Cin x Cout 72x144)
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 144, 144, 3, 1, 1, 1, 0, 0, 0, [(1, 30, 94)]),
    # hrnet-w18 f16x3 x4@960 stage3.*.branches.2.*.conv1, stage4.*.branches.2.*.conv1: Cin 72 x Cout 72 k3 s1 (the plan also runs Cin x Cout 256x24, 256x32, 256x40)
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 0, 1, 0, 3, 1, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 72, 72, 3, 1, 1, 1, 0, 0, 0, [(5, 13, 65)]),
    # r50-ga f16x3 x4@960 layer4.*.att.kv: Cin 512 x Cout 1024 k1 s2
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 0, 0, 0, 0, 0, 0, 0), 'f16x3', 'conv', 512, 1024, 1, 2, 0, 0, 0, 0, 0, [(1, 2, 2)]),
    # r50-ga f16x3 x4@960 layer3.*.att.kv: Cin 256 x Cout 512 k1 s2
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 0, 0, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 512, 1, 2, 0, 0, 0, 0, 0, [(5, 17, 33)]),
    # hrnet-w32 f16x3 x16 stage4.*.fuse_layers.1.3.0: Cin 256 x Cout 64 k1 s1
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 0, 1, 0, 0, 0, 0, 0), 'f16x3', 'conv', 256, 64, 1, 1, 1, 0, 0, 0, 0, [(1, 2, 2)]),
    # hrnet-w32 f16x3 x16 stage4.*.fuse_layers.0.3.0: Cin 256 x Cout 32 k1 s1
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 256, 32, 1, 1, 1, 0, 0, 0, 0, [(1, 2, 2)]),
    # hrnet-w18 f16x3 x4@960 stage4.*.fuse_layers.3.0.1: Cin 24 x Cout 24 k3 s2 (the plan also runs Cin x Cout 40x40)
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 1, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 24, 24, 3, 2, 1, 1, 0, 0, 0, [(5, 43, 153)]),
    # hrnet-w18 f16x3 x16/f16x3 x4@960 stage2.*.branches.0.*.conv1, stage3.*.branches.0.*.conv1, stage4.*.branches.0.*.conv1: Cin 24 x Cout 24 k3 s1 (the plan also runs Cin x Cout 32x32, 40x40, 40x72)
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 1, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 24, 24, 3, 1, 1, 1, 0, 0, 0, [(1, 133, 129)]),
    # hrnet-w18 f16x3 x4@960 stage3.*.fuse_layers.0.2.0, stage4.*.fuse_layers.0.2.0: Cin 72 x Cout 24 k1 s1 (the plan also runs Cin x Cout 72x40, 144x24, 144x40, 144x72)
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 1, 1, 1, 0, 3, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 72, 24, 1, 1, 1, 0, 0, 0, 0, [(1, 2, 2)]),
    # hrnet-w18 f16x3 x16/f16x3 x4@960 stage2.*.fuse_layers.0.1.0, stage3.*.fuse_layers.0.1.0, stage4.*.fuse_layers.0.1.0: Cin 40 x Cout 24 k1 s1 (the plan also runs Cin x Cout 64x32)
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 1, 1, 2, 0, 3, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 40, 24, 1, 1, 1, 0, 0, 0, 0, [(1, 133, 129)]),
    # r50-dcn f16x3 x16 layer3.*.c2; r50-dcnv2 f16x3 x16 layer3.*.c2: Cin 256 x Cout 256 k3 s1 (the plan also runs Cin x Cout 128x128, 512x512)
    (('f16x3', 1, 'split', 128, 1, 0, 1, 0, 0, 0, 1, 0, 2, 1, 1, 0, 0, 1, 0, 0), 'f16x3', 'deform', 256, 256, 3, 1, 1, 1, 0, 0, 0, [(4, 33, 65)]),
]


def case_id(c):
    sig, prec, kind, cin, cout, k, s = c[:7]
    d = dict(zip(SIG_FIELDS, sig))
    tags = ["BN%d" % d["BN"], "st%d" % d["stages"]]
    for f in ("ncat", "dcat", "b_resident", "epi_merge", "gn_fused"):
        if d[f]:
            tags.append(f)
    tags.append("bufs%d" % d["epi_bufs"])
    if d["residual"]:
        tags.append("res%s" % ("16" if d["residual"] == 1 else "32"))
    if d["ksplit>1"]:
        tags.append("splitk")
    tags += ["act%d" % d["relu"]] + (["bias"] if d["bias"] else []) + (["multitile"] if d["tiles>grid"] else [])
    return "%s-%s-%dx%dk%ds%d-%s" % (prec, kind, cin, cout, k, s, "-".join(tags))


def planned(c, sms=132):
    """the plan orp_tc_plan_conv reports, on a device with `sms` SMs, for the launch that test_conv_plans_gpu.Case.launch
    makes for case c: split-K where EngineTC._ksplit picks it, stem mode for stem cases, deform for deformable ones"""
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    _, prec, kind, cin, cout, k, s, bias, act, out_f32, res, gn, probs = c
    split = prec == "f16x3"
    if kind == "stem":                                     # one launch per image batch: the last one's plan
        return _lib.tc_plan_for(probs[-1:], 64, 64, 4, 1, 64, 1, 0, bias=True, relu=1, split=split, stem=2, sms=sms)
    if not split:
        cout_p = (cout + 31) // 32 * 32
    elif kind == "conv" and not out_f32 and cout <= 32:
        cout_p = 64                                        # EngineTCSplit._tc(out16=True): one 64-column TMA store tile
    else:
        cout_p = EngineTCSplit._pad_cout(cout)
    if kind == "deform":
        return _lib.tc_plan_for(probs, cout, cout_p, 3, 3, cin, 1, 1, bias=bias, relu=act, deform=True, split=split, sms=sms)
    pad = k // 2
    n, h, w = probs[0]
    L = SimpleNamespace(kh=k, kw=k, cout=cout)
    ks = EngineTC._ksplit(n, (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1, L, len(probs), act,
                          [None] if res == 1 else None, bool(out_f32), [None] if res == 2 else None)
    if ks > 1:
        return _lib.tc_plan_for(probs[:1], cout, cout_p, k, k, cin, s, pad, bias=bias, relu=act, split=split, gn=gn, ksplit=ks,
                                sms=sms)
    return _lib.tc_plan_for(probs, cout, cout_p, k, k, cin, s, pad, bias=bias, relu=act, out_f32=out_f32, split=split,
                            residual=res, gn=gn, sms=sms)
