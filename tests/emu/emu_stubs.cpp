// tests/emu/emu_stubs.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here): the pieces of the library the CPU check
// build leaves out.  The on-device BVH builder is CUB + block-synchronous kernels; the check build reports it as
// unavailable, so `gpu_bvh_build` scenes fail loudly instead of silently taking the host builder.
#include <cstdio>

#include "wbvh_gpu.h"

namespace b200pt {
bool build_wbvh_gpu(const GpuBuildInput &, cudaStream_t, GpuBuildOutput *, char *err, size_t err_len) {
    snprintf(err, err_len, "the device BVH builder is not part of the CPU check build");
    return false;
}
}  // namespace b200pt

