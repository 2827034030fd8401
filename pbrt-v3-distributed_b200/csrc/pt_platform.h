// pt_platform.h -- host/device portability shims for the path's math headers.
// The headers compile as CUDA device code in the product and as plain C++ in
// tests/host_preflight.cpp (a CPU pre-flight of the device arithmetic against
// the oracle; never linked into libb200pt.so).
#ifndef B200PT_PLATFORM_H
#define B200PT_PLATFORM_H

#include <cmath>
#include <cstdint>
#include <cstring>

// The spectrum-dependent kernels are compiled twice: RGBSpectrum (B200PT_NSPEC 3, namespace b200pt) and
// SampledSpectrum (B200PT_NSPEC 60, namespace b200pt_s60), see kernels.cu.
#ifndef B200PT_NSPEC
#define B200PT_NSPEC 3
#endif
#ifndef B200PT_NS
#define B200PT_NS b200pt
#endif

// Kernel launches go through one macro so that the CPU check build of the sources (tests/emu, -DB200PT_HOST_EMU:
// test infrastructure, see tests/emu/cuda_runtime.h) can run a kernel function once per thread index.
#define B200PT_KERNEL(...) __VA_ARGS__
#ifdef B200PT_HOST_EMU
#define B200PT_LAUNCH(kernel, grid, block, stream, ...) \
    ::b200pt_emu::launch(dim3(grid), dim3(block), [&]() { kernel(__VA_ARGS__); })
#else
#define B200PT_LAUNCH(kernel, grid, block, stream, ...) kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__)
#endif

#ifdef __CUDACC__
#define B200_HD __host__ __device__ __forceinline__
#define B200_D __device__ __forceinline__
#else
#define B200_HD inline
#define B200_D inline
#endif
// Everything above is force-inlined, which made the shading kernels 18-55 k instructions long; profiling showed their
// warps waiting for instruction fetches.  B200PT_OUTLINE >= 1 keeps one copy of the BSDF entry points
// (bsdf_f / bsdf_pdf / bsdf_sample_f), >= 2 also of the lobe functions and the microfacet sampling routine.  Inlining never changes a result bit (no contraction, no fast math).
// Level 1 measured fastest of the three when it was chosen and is the default; not re-measured on the H100.
#ifndef B200PT_OUTLINE
#define B200PT_OUTLINE 1
#endif
#if defined(__CUDACC__) && B200PT_OUTLINE >= 1
#define B200_HD_L1 inline __host__ __device__ __noinline__
#else
#define B200_HD_L1 B200_HD
#endif
#if defined(__CUDACC__) && B200PT_OUTLINE >= 2
#define B200_HD_L2 inline __host__ __device__ __noinline__
#else
#define B200_HD_L2 B200_HD
#endif
#if defined(__CUDACC__) && defined(B200PT_S60_OUTLINE)
#define B200_HD_S60 inline __host__ __device__ __noinline__
#else
#define B200_HD_S60 B200_HD
#endif

namespace B200PT_NS {

B200_HD uint32_t float_as_uint(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
#endif
}
B200_HD float uint_as_float(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}

}  // namespace B200PT_NS
#endif
