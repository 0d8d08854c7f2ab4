"""Compile the reference's CARAFE naive forward kernel (mmdet/ops/carafe/src/carafe_naive_cuda_kernel.cu,
CARAFENAIVEForward) as host C++ into oracle/_ref/ref_carafe_naive_dev.so, through build_ref._device_as_host: the part of
the .cu file above its host launchers, read where it lies and piped to g++ with oracle/ref_harness_carafe_device.inc
(TEST INFRASTRUCTURE).  Only runs where the reference's source tree exists; elsewhere build() returns None."""
import os

from .build_ref import HERE, OUT, REF, _device_as_host

# the grid-stride loop of CUDA_1D_KERNEL_LOOP runs every index on the host with one thread in one block; GET_BLOCKS uses min
_PREFIX = ("namespace at {}\nusing std::min;\nstruct uint3_ { unsigned x, y, z; };\n"
           "static uint3_ blockIdx = {0, 0, 0}, threadIdx = {0, 0, 0}, blockDim = {1, 1, 1}, gridDim = {1, 1, 1};\n")


def build(verbose=False):
    if not os.path.isdir(REF):
        return None
    os.makedirs(OUT, exist_ok=True)
    out = os.path.join(OUT, "ref_carafe_naive_dev.so")
    _device_as_host(os.path.join(REF, "mmdet/ops/carafe/src/carafe_naive_cuda_kernel.cu"), "int CARAFENAIVEForwardLaucher",
                    os.path.join(HERE, "ref_harness_carafe_device.inc"), out, verbose, _PREFIX)
    return out if os.path.exists(out) else None


if __name__ == "__main__":
    print(build(verbose=True))
