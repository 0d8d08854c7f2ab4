"""Compile the reference's own CPU sources of the path into oracle/_ref/ (TEST INFRASTRUCTURE).

Sources are compiled FROM WHERE THEY LIE in the reference's source tree, $ORP_REFERENCE_ROOT (nothing is copied
into the repo; oracle/_ref/ is git-ignored).

  libref_polyiou.so   DOTA_devkit/polyiou.cpp  (+ oracle/ref_harness_polyiou.cpp, C ABI re-export)
  _polyiou<EXT>.so    DOTA_devkit/polyiou_wrap.cxx + polyiou.cpp  (the reference's SWIG module;
                      polyiou.py is copied next to it as a build OUTPUT so `import polyiou` works)
  ref_rnms_cpu.so     mmdet/ops/nms/src/rnms_cpu.cpp unmodified (+ oracle/ref_harness_rnms.cpp)
  ref_box_iou_rotated.so  mmdet/ops/box_iou_rotated/src/box_iou_rotated_cpu.cpp unmodified

  ref_minarearect_dev.so / ref_convex_iou_dev.so / ref_poly_nms_dev.so / ref_poly_overlaps_dev.so
                      the __device__ functions of minarearect_kernel.cu / convex_iou_kernel.cu / poly_nms_kernel.cu / poly_overlaps_kernel.cu
  ref_dcn_dev.so      deform_conv_cuda_kernel.cu: bilinear samplers + the (modulated_)deformable_im2col KERNELS run on the host
                      compiled as HOST C++ (the text above their __global__ kernel, piped to g++; see _device_as_host)

Only runs where that tree exists; elsewhere build() returns None.  The reference's CUDA
sources (mmdet/ops/**/src/*.cu) are NOT buildable as CUDA: they include THC/THC.h which torch 2.11
no longer ships (SURVEY.md section 8c) - stated in DESIGN.md.
"""
import os
import shutil
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = os.environ.get("ORP_REFERENCE_ROOT", "/root/reference")


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)


def _stale(target, deps):
    return (not os.path.exists(target)) or any(os.path.getmtime(target) < os.path.getmtime(d) for d in deps)


_DEVICE_PREFIX = """
#define __device__
#define __host__
#define __global__
#include <math.h>
#include <stdio.h>
#include <algorithm>
#include <vector>
"""


def _device_as_host(cu_path, cut_marker, wrapper_path, out_so, verbose, extra_prefix=""):
    """compile the part of a reference .cu file that precedes `cut_marker` (its __device__ functions) as host C++"""
    if not (os.path.exists(cu_path) and os.path.exists(wrapper_path)):
        return
    if not _stale(out_so, [cu_path, wrapper_path, os.path.abspath(__file__)]):
        return
    text = open(cu_path).read()
    if isinstance(cut_marker, str):
        segments = [(None, cut_marker)]
    else:
        segments = cut_marker                       # [(start marker or None, end marker), ...]: several device-only ranges
    part = ""
    for a, b in segments:
        i0 = 0 if a is None else text.index(a)
        part += text[i0:text.index(b, i0)] + "\n"
    body = "\n".join(l for l in part.splitlines() if not l.lstrip().startswith("#include"))   # ATen / THC headers
    unit = _DEVICE_PREFIX + extra_prefix + body + "\n" + open(wrapper_path).read()
    cmd = ["g++", "-x", "c++", "-", "-O2", "-shared", "-fPIC", "-w", "-ffp-contract=off", "-o", out_so]
    if verbose:
        print(" ".join(cmd), "  <", cu_path, "(device part) +", wrapper_path)
    subprocess.run(cmd, input=unit.encode(), check=True)


def build(verbose=False, with_torch=True):
    if not os.path.isdir(REF):
        return None
    os.makedirs(OUT, exist_ok=True)
    devkit = os.path.join(REF, "DOTA_devkit")
    # 1. polyiou.cpp behind a C ABI
    lib = os.path.join(OUT, "libref_polyiou.so")
    harness = os.path.join(HERE, "ref_harness_polyiou.cpp")
    src = os.path.join(devkit, "polyiou.cpp")
    if _stale(lib, [harness, src]):
        _run(["g++", "-O2", "-shared", "-fPIC", "-w", '-DREF_POLYIOU_CPP="%s"' % src, harness, "-o", lib], verbose)
    # 2. the SWIG module exactly as the reference ships it (checked-in wrapper, no swig needed)
    ext = sysconfig.get_config_var("EXT_SUFFIX")
    swig = os.path.join(OUT, "_polyiou" + ext)
    wrap = os.path.join(devkit, "polyiou_wrap.cxx")
    if _stale(swig, [wrap, src]):
        _run(["g++", "-O2", "-shared", "-fPIC", "-w", "-I" + sysconfig.get_paths()["include"],
              "-I" + devkit, wrap, src, "-o", swig], verbose)
        shutil.copyfile(os.path.join(devkit, "polyiou.py"), os.path.join(OUT, "polyiou.py"))
    # 2b. the DEVICE functions of the reference's CUDA-only ops, compiled as host C++.  The .cu files cannot be built as
    #     CUDA (THC headers), but everything above their __global__ kernel is plain C++ behind `__device__`: that part is
    #     piped to g++ (read where it lies, cut at the kernel, never written to disk) between a prefix that blanks the
    #     CUDA qualifiers / missing headers and a C-ABI wrapper.  -ffp-contract=off: separately rounded operations.
    _device_as_host(os.path.join(REF, "mmdet/ops/minarearect/src/minarearect_kernel.cu"), "__global__ void minareabbox_kernel",
                    os.path.join(HERE, "ref_harness_minarearect_device.inc"), os.path.join(OUT, "ref_minarearect_dev.so"), verbose)
    _device_as_host(os.path.join(REF, "mmdet/ops/iou/src/convex_iou_kernel.cu"), "__global__ void convex_iou_kernel",
                    os.path.join(HERE, "ref_harness_convex_iou_device.inc"), os.path.join(OUT, "ref_convex_iou_dev.so"), verbose)
    f2 = ("struct float2 { float x, y; };\nstatic inline float2 make_float2(float x, float y) { float2 r; r.x = x; r.y = y; return r; }\n"
          "struct uint3_ { unsigned x, y, z; };\nstatic uint3_ blockIdx, blockDim, threadIdx;   // referenced by leftover debug code\n")
    _device_as_host(os.path.join(devkit, "poly_nms_gpu/poly_nms_kernel.cu"), "__global__ void poly_nms_kernel",
                    os.path.join(HERE, "ref_harness_poly_nms_device.inc"), os.path.join(OUT, "ref_poly_nms_dev.so"), verbose, f2)
    _device_as_host(os.path.join(devkit, "poly_nms_gpu/poly_overlaps_kernel.cu"), "__global__ void overlaps_kernel",
                    os.path.join(HERE, "ref_harness_poly_overlaps_device.inc"), os.path.join(OUT, "ref_poly_overlaps_dev.so"), verbose, f2)
    # DCN: the bilinear sampler + the im2col KERNELS themselves (their grid-stride loop macro runs the whole index range on the
    # host once blockIdx = threadIdx = 0 and blockDim = gridDim = 1); DCNv1 range + DCNv2 (modulated) range of the file
    cuda1 = ("namespace at {}\nstruct uint3_ { unsigned x, y, z; };\n"
             "static uint3_ blockIdx = {0, 0, 0}, threadIdx = {0, 0, 0}, blockDim = {1, 1, 1}, gridDim = {1, 1, 1};\n")
    _device_as_host(os.path.join(REF, "mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu"),
                    [(None, "void deformable_im2col("),
                     ("template <typename scalar_t>\n__device__ scalar_t dmcn_im2col_bilinear", "template <typename scalar_t>\n__device__ scalar_t dmcn_get_gradient_weight"),
                     ("template <typename scalar_t>\n__global__ void modulated_deformable_im2col_gpu_kernel",
                      "template <typename scalar_t>\n__global__ void modulated_deformable_col2im_gpu_kernel")],
                    os.path.join(HERE, "ref_harness_dcn_device.inc"), os.path.join(OUT, "ref_dcn_dev.so"), verbose, cuda1)
    if not with_torch:
        return OUT
    # 3./4. torch CPU extensions, reference sources unmodified
    import torch  # noqa: F401
    from torch.utils import cpp_extension as ce
    inc = []
    for p in ce.include_paths():
        inc += ["-isystem", p]
    inc += ["-I" + sysconfig.get_paths()["include"]]
    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    common = ["g++", "-O2", "-shared", "-fPIC", "-w", "-std=c++17",
              "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)] + inc
    link = ["-L" + tlib, "-Wl,-rpath," + tlib, "-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python"]
    rn = os.path.join(OUT, "ref_rnms_cpu.so")
    rsrc = os.path.join(REF, "mmdet/ops/nms/src/rnms_cpu.cpp")
    rh = os.path.join(HERE, "ref_harness_rnms.cpp")
    if _stale(rn, [rsrc, rh]):
        _run(common + ["-DTORCH_EXTENSION_NAME=ref_rnms_cpu", rsrc, rh, "-o", rn] + link, verbose)
    bi = os.path.join(OUT, "ref_box_iou_rotated.so")
    bsrc = os.path.join(REF, "mmdet/ops/box_iou_rotated/src/box_iou_rotated_cpu.cpp")
    bh = os.path.join(HERE, "ref_harness_box_iou_rotated.cpp")
    if os.path.exists(bh) and _stale(bi, [bsrc, bh]):
        _run(common + ["-I" + os.path.dirname(bsrc), bsrc, bh, "-o", bi] + link, verbose)
    return OUT


if __name__ == "__main__":
    print(build(verbose=True))
