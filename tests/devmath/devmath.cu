// tests/devmath/devmath.cu -- TEST INFRASTRUCTURE: evaluates the path's scalar math on the device, as nvcc compiles it
// for the product (same headers, same flags: csrc/nvflags.mk), and compares it bit for bit with the host's glibc (the
// calls the reference makes) or with the host-compiled build of the same headers.  Loaded by tests/test_zz_devmath_gpu.py
// (and, without a device, by tests/test_devmath.py for its host half) through ctypes.
// Its texture half runs ImageTexture's MIPMap lookups, RoughnessToAlpha, InfiniteAreaLight's Le / Sample_Li / Pdf_Li
// (pt_texture.cuh) and ComputeDifferentials (pt_core.cuh) on the device or host-compiled, over tables and queries the
// reference's own classes answered (oracle/probe/ref_probe.cpp), for tests/test_zz_texlookup_gpu.py and
// tests/test_texlookup.py.
//
// Pass rule: equal bits, or both outputs NaN (NaN payloads legitimately differ between the device and x86).
// Device work goes in chunks of at most 256 MiB of outputs, and every call frees what it allocated.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <thread>
#include <vector>

#include "pt_sphere.cuh"
#if __has_include("pt_texture.cuh")
#include "pt_texture.cuh"
#define DM_TEXTURE 1
#endif

using namespace b200pt;

// The double cos / sin tr_sample11 calls: the restatement, or libdevice's when built against headers that predate it
// (which is how the harness measures what the restatement fixes).
#if __has_include("pt_sincos_dbl.cuh")
#define DM_COS pt_cos
#define DM_SIN pt_sin
#else
#define DM_COS ::cos
#define DM_SIN ::sin
#endif

enum {
    DM_EXPF = 0, DM_LOGF, DM_SINF, DM_COSF, DM_ACOSF, DM_ATANF,  // float f(float) over bit patterns start + i
    DM_PHI_COS, DM_PHI_SIN,                                       // double f((double)phi(U2)) over U2 = bits start + i
    DM_ATAN2F,                                                    // float atan2f(y, x) over pairs
    DM_NFUNC
};
enum { DM_REF_GLIBC = 0, DM_REF_HOST = 1 };

extern "C" struct dm_report {
    uint64_t checked, mismatches;
    int32_t n_first, pad;
    uint64_t input[16];  // bit pattern, U2 bits, (y bits << 32 | x bits), or (point << 3 | output word)
    uint64_t got[16], want[16];
};

static const uint64_t CHUNK_BYTES = 256ull << 20;

// ---------------------------------------------------------------------------------------------------- inputs
B200_HD float phi_of(float U2) { return (float)(6.28318530718 * (double)U2); }  // tr_sample11, pt_core.cuh
B200_HD uint64_t splitmix64(uint64_t z) {
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
// Pair k of the random atan2f set: even k any two bit patterns, odd k two floats in [-3, 3).
B200_HD void random_pair(uint64_t seed, uint64_t k, float *y, float *x) {
    const uint64_t h = splitmix64(seed * 0x100000001b3ull + k);
    if (k & 1) {
        *y = (float)(h & 0xffffffu) * 0x1p-24f * 6.f - 3.f;
        *x = (float)((h >> 32) & 0xffffffu) * 0x1p-24f * 6.f - 3.f;
    } else {
        *y = uint_as_float((uint32_t)h);
        *x = uint_as_float((uint32_t)(h >> 32));
    }
}

// ---------------------------------------------------------------------------------------------------- device side
template <int F>
__global__ void k_unary(uint64_t start, uint64_t n, void *out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = uint_as_float((uint32_t)(start + i));
    if (F == DM_PHI_COS || F == DM_PHI_SIN) {
        const double p = (double)phi_of(x);
        ((uint64_t *)out)[i] = double_as_u64(F == DM_PHI_COS ? DM_COS(p) : DM_SIN(p));
        return;
    }
    float r = 0.f;
    switch (F) {
    case DM_EXPF: r = pt_expf(x); break;
    case DM_LOGF: r = pt_logf(x); break;
    case DM_SINF: r = pt_sinf(x); break;
    case DM_COSF: r = pt_cosf(x); break;
    case DM_ACOSF: r = pt_acosf(x); break;
    case DM_ATANF: r = pt_atanf(x); break;
    }
    ((uint32_t *)out)[i] = float_as_uint(r);
}

__global__ void k_atan2(const float *ys, const float *xs, uint64_t seed, uint64_t start, uint64_t n, uint32_t *out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float y, x;
    if (ys) {
        y = ys[start + i];
        x = xs[start + i];
    } else {
        random_pair(seed, start + i, &y, &x);
    }
    out[i] = float_as_uint(pt_atan2f(y, x));
}

// ---------------------------------------------------------------------------------------------------- composites
// Sampling helpers evaluated at grid points (u0, u1) = (ax[i % nx], ay[i / nx]); each writes DM_WORDS output words
// (unused ones stay 0).  params: per-helper constants, see the cases.
enum {
    DM_C_DISK = 0, DM_C_HG, DM_C_TR11, DM_C_TR_WH, DM_C_SPHDIR, DM_C_SPH_AREA, DM_C_SPH_CONE, DM_C_DISCRETE,
    DM_C_HALTON, DM_NCOMP
};
#define DM_WORDS 8

B200_HD DevSphere dm_sphere(const float *c, float radius) {
    DevSphere s;
    memset(&s, 0, sizeof(s));
    for (int i = 0; i < 4; ++i) s.o2w[5 * i] = s.w2o[5 * i] = 1.f;
    for (int a = 0; a < 3; ++a) {
        s.o2w[4 * a + 3] = c[a];
        s.w2o[4 * a + 3] = -c[a];
    }
    s.radius = radius;
    s.phi_max = 2 * PT_PI;
    s.theta_min = PT_PI;
    s.z_min = -radius;
    s.z_max = radius;
    s.area = s.phi_max * radius * (s.z_max - s.z_min);
    return s;
}

B200_HD void composite_eval(int which, const float *prm, float u0, float u1, uint32_t *o) {
    float f[DM_WORDS] = {0, 0, 0, 0, 0, 0, 0, 0};
    const float u[2] = {u0, u1};
    switch (which) {
    case DM_C_DISK:  // concentric_sample_disk
        concentric_sample_disk(u, f);
        break;
    case DM_C_HG: {  // hg_sample_p(g = prm[0], wo = normalize(prm[1..3]))
        V3 wi;
        f[3] = hg_sample_p(prm[0], normalize(mk(prm[1], prm[2], prm[3])), &wi, u);
        f[0] = wi.x, f[1] = wi.y, f[2] = wi.z;
        break;
    }
    case DM_C_TR11:  // tr_sample11(cosTheta = prm[0], U1 = u0, U2 = u1)
        tr_sample11(prm[0], u0, u1, &f[0], &f[1]);
        break;
    case DM_C_TR_WH: {  // tr_sample_wh({prm[0], prm[1]}, wo = normalize(prm[2..4]))
        TRDist d;
        d.ax = prm[0], d.ay = prm[1];
        const V3 wh = tr_sample_wh(d, normalize(mk(prm[2], prm[3], prm[4])), u);
        f[0] = wh.x, f[1] = wh.y, f[2] = wh.z;
        break;
    }
    case DM_C_SPHDIR: {  // spherical_direction(uniform-sphere cosTheta of u0, phi = 2 pi u1, frame of prm[0..2])
        const float cosTheta = 1 - 2 * u0, sinTheta = sqrtf(pt_max(0.f, 1 - cosTheta * cosTheta));
        V3 z = normalize(mk(prm[0], prm[1], prm[2])), x, y;
        coordinate_system(z, &x, &y);
        const V3 w = spherical_direction(sinTheta, cosTheta, 2 * PT_PI * u1, x, y, z);
        f[0] = w.x, f[1] = w.y, f[2] = w.z;
        break;
    }
    case DM_C_SPH_AREA:    // sphere_sample_area(centre prm[0..2], radius prm[3])
    case DM_C_SPH_CONE: {  // sphere_sample from prm[4..6] (outside the sphere: the cone branch)
        const DevSphere s = dm_sphere(prm, prm[3]);
        const V3 zero = mk(0.f, 0.f, 0.f);
        const LightSample ls = which == DM_C_SPH_AREA ? sphere_sample_area(s, u, &f[6])
                                                      : sphere_sample(s, mk(prm[4], prm[5], prm[6]), zero, zero, u, &f[6]);
        f[0] = ls.p.x, f[1] = ls.p.y, f[2] = ls.p.z, f[3] = ls.n.x, f[4] = ls.n.y, f[5] = ls.n.z;
        break;
    }
    case DM_C_DISCRETE: {  // sample_discrete over {0, 1, 0, 3, 0.5, 2, 0, 0.25} (Distribution1D's cdf) at u0 and u1
        const int n = 8;
        const float func[n] = {0.f, 1.f, 0.f, 3.f, 0.5f, 2.f, 0.f, 0.25f};
        float cdf[n + 1];
        cdf[0] = 0;
        for (int i = 1; i <= n; ++i) cdf[i] = cdf[i - 1] + func[i - 1] / n;
        const float funcInt = cdf[n];
        for (int i = 1; i <= n; ++i) cdf[i] /= funcInt;
        f[0] = (float)sample_discrete(cdf, func, funcInt, n, u0, &f[1]);
        f[2] = (float)sample_discrete(cdf, func, funcInt, n, u1, &f[3]);
        break;
    }
    case DM_C_HALTON: {  // halton_radical_inverse(base prm[0], a = bits(u0) << 32 | bits(u1)), plain and permuted
        const uint32_t base = (uint32_t)prm[0];
        uint16_t perm[64];
        // d -> 5d + 3 mod base permutes the digits of every base the tests use (3, 7, 61: all prime to 5)
        for (uint32_t d = 0; d < base && d < 64; ++d) perm[d] = (uint16_t)((d * 5 + 3) % base);
        const uint64_t a = ((uint64_t)float_as_uint(u0) << 32) | float_as_uint(u1);
        f[0] = halton_radical_inverse(base, nullptr, a);
        f[1] = halton_radical_inverse(base, perm, a);
        f[2] = halton_radical_inverse(base, nullptr, a >> 32);
        break;
    }
    }
    for (int w = 0; w < DM_WORDS; ++w) o[w] = float_as_uint(f[w]);
}

struct DmParams {
    float p[8];
};
__global__ void k_composite(int which, DmParams prm, const float *ax, uint64_t nx, const float *ay, uint64_t start,
                            uint64_t n, uint32_t *out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t k = start + i;
    composite_eval(which, prm.p, ax[k % nx], ay[k / nx], out + i * DM_WORDS);
}

// ---------------------------------------------------------------------------------------------------- host side
template <class Fn>
static void parallel_for(uint64_t n, Fn fn) {
    const unsigned nt = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
    std::vector<std::thread> pool;
    const uint64_t per = (n + nt - 1) / nt;
    for (unsigned t = 0; t < nt; ++t) {
        const uint64_t lo = std::min(n, t * per), hi = std::min(n, lo + per);
        pool.emplace_back([=]() { fn(lo, hi); });
    }
    for (auto &th : pool) th.join();
}

// one function per loop, so that the compiler cannot pair sin and cos into sincos (also -fno-builtin-sin/-cos)
template <int F>
static void host_unary(int ref, uint64_t start, uint64_t n, void *out) {
    parallel_for(n, [=](uint64_t lo, uint64_t hi) {
        for (uint64_t i = lo; i < hi; ++i) {
            const float x = uint_as_float((uint32_t)(start + i));
            if (F == DM_PHI_COS || F == DM_PHI_SIN) {
                const double p = (double)phi_of(x);
                double r;
                if (F == DM_PHI_COS)
                    r = ref == DM_REF_GLIBC ? ::cos(p) : DM_COS(p);
                else
                    r = ref == DM_REF_GLIBC ? ::sin(p) : DM_SIN(p);
                ((uint64_t *)out)[i] = double_as_u64(r);
                continue;
            }
            float r = 0.f;
            const bool g = ref == DM_REF_GLIBC;
            switch (F) {
            case DM_EXPF: r = g ? std::exp(x) : pt_expf(x); break;
            case DM_LOGF: r = g ? std::log(x) : pt_logf(x); break;
            case DM_SINF: r = g ? std::sin(x) : pt_sinf(x); break;
            case DM_COSF: r = g ? std::cos(x) : pt_cosf(x); break;
            case DM_ACOSF: r = g ? std::acos(x) : pt_acosf(x); break;
            case DM_ATANF: r = g ? std::atan(x) : pt_atanf(x); break;
            }
            ((uint32_t *)out)[i] = float_as_uint(r);
        }
    });
}

static bool is_wide(int f) { return f == DM_PHI_COS || f == DM_PHI_SIN; }

static bool nan_bits(uint64_t v, bool wide) {
    return wide ? ((v & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) : ((v & 0x7fffffffu) > 0x7f800000u);
}

extern "C" {

// Evaluates a unary function on the host: glibc (ref 0) or the host-compiled restatement (ref 1).  out holds n 32-bit
// words, or n 64-bit words for DM_PHI_COS / DM_PHI_SIN.
int dm_host_unary(int f, int ref, uint64_t start, uint64_t n, void *out) {
    switch (f) {
    case DM_EXPF: host_unary<DM_EXPF>(ref, start, n, out); break;
    case DM_LOGF: host_unary<DM_LOGF>(ref, start, n, out); break;
    case DM_SINF: host_unary<DM_SINF>(ref, start, n, out); break;
    case DM_COSF: host_unary<DM_COSF>(ref, start, n, out); break;
    case DM_ACOSF: host_unary<DM_ACOSF>(ref, start, n, out); break;
    case DM_ATANF: host_unary<DM_ATANF>(ref, start, n, out); break;
    case DM_PHI_COS: host_unary<DM_PHI_COS>(ref, start, n, out); break;
    case DM_PHI_SIN: host_unary<DM_PHI_SIN>(ref, start, n, out); break;
    default: return -1;
    }
    return 0;
}

// Compares got with want (wide: 64-bit words) and adds to the report; input of element i is input_base + i * input_step.
void dm_compare(const void *got, const void *want, uint64_t n, int wide, uint64_t input_base, uint64_t input_step,
                dm_report *rep) {
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t g = wide ? ((const uint64_t *)got)[i] : ((const uint32_t *)got)[i];
        const uint64_t w = wide ? ((const uint64_t *)want)[i] : ((const uint32_t *)want)[i];
        if (g == w || (nan_bits(g, wide) && nan_bits(w, wide))) continue;
        if (rep->n_first < 16) {
            rep->input[rep->n_first] = input_base + i * input_step;
            rep->got[rep->n_first] = g;
            rep->want[rep->n_first] = w;
            rep->n_first++;
        }
        rep->mismatches++;
    }
    rep->checked += n;
}

static int cuda_fail(cudaError_t e, const char *what) {
    fprintf(stderr, "devmath: %s: %s\n", what, cudaGetErrorString(e));
    return -(int)e - 1000;
}
#define DM_CUDA(call)                                        \
    do {                                                     \
        cudaError_t e_ = (call);                             \
        if (e_ != cudaSuccess) {                             \
            rc = cuda_fail(e_, #call);                       \
            goto done;                                       \
        }                                                    \
    } while (0)

// Device function f at bit patterns [start, end) against the host (ref: glibc or host-compiled restatement).
int dm_check_unary(int f, int ref, uint64_t start, uint64_t end, dm_report *rep) {
    if (f < 0 || f >= DM_ATAN2F || end < start) return -1;
    const bool wide = is_wide(f);
    const uint64_t word = wide ? 8 : 4, chunk = std::max<uint64_t>(1, std::min(CHUNK_BYTES / word, end - start));
    std::vector<uint8_t> hd(chunk * word), hh(chunk * word);
    void *d = nullptr;
    int rc = 0;
    DM_CUDA(cudaMalloc(&d, chunk * word));
    for (uint64_t s = start; s < end; s += chunk) {
        const uint64_t n = std::min(chunk, end - s);
        const unsigned blocks = (unsigned)((n + 255) / 256);
        switch (f) {
        case DM_EXPF: k_unary<DM_EXPF><<<blocks, 256>>>(s, n, d); break;
        case DM_LOGF: k_unary<DM_LOGF><<<blocks, 256>>>(s, n, d); break;
        case DM_SINF: k_unary<DM_SINF><<<blocks, 256>>>(s, n, d); break;
        case DM_COSF: k_unary<DM_COSF><<<blocks, 256>>>(s, n, d); break;
        case DM_ACOSF: k_unary<DM_ACOSF><<<blocks, 256>>>(s, n, d); break;
        case DM_ATANF: k_unary<DM_ATANF><<<blocks, 256>>>(s, n, d); break;
        case DM_PHI_COS: k_unary<DM_PHI_COS><<<blocks, 256>>>(s, n, d); break;
        case DM_PHI_SIN: k_unary<DM_PHI_SIN><<<blocks, 256>>>(s, n, d); break;
        }
        DM_CUDA(cudaGetLastError());
        dm_host_unary(f, ref, s, n, hh.data());  // overlaps the kernel
        DM_CUDA(cudaMemcpy(hd.data(), d, n * word, cudaMemcpyDeviceToHost));
        dm_compare(hd.data(), hh.data(), n, wide, s, 1, rep);
    }
done:
    cudaFree(d);
    return rc;
}

// Host atan2f over pairs: explicit (ys, xs non-null, elements [start, start + n)) or random (pair k = random_pair(seed, k)).
int dm_host_atan2(int ref, const float *ys, const float *xs, uint64_t seed, uint64_t start, uint64_t n, uint32_t *out) {
    parallel_for(n, [=](uint64_t lo, uint64_t hi) {
        for (uint64_t i = lo; i < hi; ++i) {
            float y, x;
            if (ys) {
                y = ys[start + i];
                x = xs[start + i];
            } else {
                random_pair(seed, start + i, &y, &x);
            }
            out[i] = float_as_uint(ref == DM_REF_GLIBC ? std::atan2(y, x) : pt_atan2f(y, x));
        }
    });
    return 0;
}

// Device atan2f against the host over n pairs (explicit when ys / xs are given, random from seed otherwise).  The report's
// input is (y bits << 32) | x bits.
int dm_check_atan2(int ref, const float *ys, const float *xs, uint64_t seed, uint64_t n, dm_report *rep) {
    const uint64_t chunk = std::max<uint64_t>(1, std::min(CHUNK_BYTES / 4, n));
    std::vector<uint32_t> hd(chunk), hh(chunk);
    uint32_t *d = nullptr;
    float *dy = nullptr, *dx = nullptr;
    int rc = 0;
    DM_CUDA(cudaMalloc(&d, chunk * 4));
    if (ys) {
        DM_CUDA(cudaMalloc(&dy, n * 4));
        DM_CUDA(cudaMalloc(&dx, n * 4));
        DM_CUDA(cudaMemcpy(dy, ys, n * 4, cudaMemcpyHostToDevice));
        DM_CUDA(cudaMemcpy(dx, xs, n * 4, cudaMemcpyHostToDevice));
    }
    for (uint64_t s = 0; s < n; s += chunk) {
        const uint64_t m = std::min(chunk, n - s);
        k_atan2<<<(unsigned)((m + 255) / 256), 256>>>(dy, dx, seed, s, m, d);
        DM_CUDA(cudaGetLastError());
        dm_host_atan2(ref, ys, xs, seed, s, m, hh.data());
        DM_CUDA(cudaMemcpy(hd.data(), d, m * 4, cudaMemcpyDeviceToHost));
        const uint64_t before = rep->n_first;
        dm_compare(hd.data(), hh.data(), m, 0, s, 1, rep);
        for (uint64_t j = before; j < (uint64_t)rep->n_first; ++j) {  // pair index -> the pair's bits
            float y, x;
            const uint64_t k = rep->input[j];
            if (ys) {
                y = ys[k];
                x = xs[k];
            } else {
                random_pair(seed, k, &y, &x);
            }
            rep->input[j] = ((uint64_t)float_as_uint(y) << 32) | float_as_uint(x);
        }
    }
done:
    cudaFree(d);
    cudaFree(dy);
    cudaFree(dx);
    return rc;
}

// Host composite helper at grid points [start, start + n): DM_WORDS words per point.
int dm_host_composite(int which, const float *params, const float *ax, uint64_t nx, const float *ay, uint64_t start,
                      uint64_t n, uint32_t *out) {
    if (which < 0 || which >= DM_NCOMP) return -1;
    parallel_for(n, [=](uint64_t lo, uint64_t hi) {
        for (uint64_t i = lo; i < hi; ++i) {
            const uint64_t k = start + i;
            composite_eval(which, params, ax[k % nx], ay[k / nx], out + i * DM_WORDS);
        }
    });
    return 0;
}

// Device composite helper against the host-compiled build at the nx * ny grid points; the report's input is
// (point << 3) | word.  With got non-null, also returns the device's words for the first min(ngot, nx * ny) points.
int dm_check_composite(int which, const float *params, const float *ax, uint64_t nx, const float *ay, uint64_t ny,
                       dm_report *rep, uint32_t *got, uint64_t ngot) {
    if (which < 0 || which >= DM_NCOMP) return -1;
    const uint64_t total = nx * ny, chunk = std::max<uint64_t>(1, std::min(CHUNK_BYTES / (4 * DM_WORDS), total));
    std::vector<uint32_t> hd(chunk * DM_WORDS), hh(chunk * DM_WORDS);
    DmParams prm;
    for (int i = 0; i < 8; ++i) prm.p[i] = params[i];
    uint32_t *d = nullptr;
    float *dax = nullptr, *day = nullptr;
    int rc = 0;
    DM_CUDA(cudaMalloc(&d, chunk * DM_WORDS * 4));
    DM_CUDA(cudaMalloc(&dax, nx * 4));
    DM_CUDA(cudaMalloc(&day, ny * 4));
    DM_CUDA(cudaMemcpy(dax, ax, nx * 4, cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(day, ay, ny * 4, cudaMemcpyHostToDevice));
    for (uint64_t s = 0; s < total; s += chunk) {
        const uint64_t m = std::min(chunk, total - s);
        k_composite<<<(unsigned)((m + 255) / 256), 256>>>(which, prm, dax, nx, day, s, m, d);
        DM_CUDA(cudaGetLastError());
        dm_host_composite(which, params, ax, nx, ay, s, m, hh.data());
        DM_CUDA(cudaMemcpy(hd.data(), d, m * DM_WORDS * 4, cudaMemcpyDeviceToHost));
        dm_compare(hd.data(), hh.data(), m * DM_WORDS, 0, s * DM_WORDS, 1, rep);
        if (got && s < ngot) std::copy(hd.begin(), hd.begin() + std::min(m, ngot - s) * DM_WORDS, got + s * DM_WORDS);
    }
done:
    cudaFree(d);
    cudaFree(dax);
    cudaFree(day);
    return rc;
}

}  // extern "C"

#ifdef DM_TEXTURE
// ---------------------------------------------------------------------------------------------------- textures and sky
// One query per thread.  Query floats and answer words of each family:
//   DM_T_EWA     {s, t, dst0.x, dst0.y, dst1.x, dst1.y} -> Lookup(st, dst0, dst1): r, g, b
//   DM_T_WIDTH   {s, t, width}                          -> Lookup(st, width): r, g, b
//   DM_T_SAMPLE  {u0, u1}                               -> Sample_Li: wi[3], pdf, Li[3], the visibility target[3]
//   DM_T_PDF     {w[3]}                                 -> Pdf_Li
//   DM_T_LE      {ray.d[3]}                             -> Le: r, g, b
//   DM_T_DIFF    {p, n, dpdu, dpdv, rxOrigin, rxDirection, ryOrigin, ryDirection} -> dudx, dvdx, dudy, dvdy
//   DM_T_ROUGH   {roughness}                            -> RoughnessToAlpha
// A float MIPMap is uploaded as (v, v, v, 0) like b200pt_scene_add_mipmap does; its answers are compared on all three words.
enum { DM_T_EWA = 0, DM_T_WIDTH, DM_T_SAMPLE, DM_T_PDF, DM_T_LE, DM_T_DIFF, DM_T_ROUGH, DM_T_N };
static const int DM_T_IN[DM_T_N] = {6, 3, 2, 3, 3, 24, 1};
static const int DM_T_OUT[DM_T_N] = {3, 3, 10, 1, 3, 4, 1};
enum { DM_ON_HOST = 0, DM_ON_DEVICE = 1 };
// The largest EWA bounding box (texels) a query may scan, and the largest |st * size| it may reach: beyond 2^31 the
// device's (int)ceilf saturates where x86 gives INT_MIN, and a box ending at INT_MAX never ends (DESIGN.md, limits)
#define DM_EWA_MAX_TEXELS 4096
#define DM_ST_MAX 1073741824.f

// The tables, as ref_probe returned them.  Levels: [h][w][channels] each, one after the other.
extern "C" struct dm_mipmap {
    int32_t channels, levels, wrap, trilinear;
    float max_aniso;
    int32_t w[B200PT_MIPMAP_MAX_LEVELS], h[B200PT_MIPMAP_MAX_LEVELS];
    const float *texels;
    float weight_lut[128];
};
extern "C" struct dm_sky {
    int32_t w, h, nu, nv;
    const float *texels;  // [h][w][3]
    const float *cond_func, *cond_cdf, *cond_func_int, *marg_func, *marg_cdf;
    float marg_func_int;
    float light_to_world[16], world_to_light[16];
    float two_world_radius;
    float ref_p[3];
};

struct TexCtx {
    DevMipmap M;
    DevInfinite L;
    float ref_p[3];
};

B200_HD void tex_eval(const TexCtx &c, int fam, const float *q, int nout, uint32_t *o) {
    float f[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    switch (fam) {
    case DM_T_EWA:
    case DM_T_WIDTH: {
        const Spec v = fam == DM_T_EWA ? mip_lookup(c.M, q[0], q[1], q[2], q[3], q[4], q[5]) : mip_lookup_width(c.M, q[0], q[1], q[2]);
        f[0] = v.c[0], f[1] = v.c[1], f[2] = v.c[2];
        break;
    }
    case DM_T_SAMPLE: {
        V3 wi, pt;
        float pdf;
        const Spec li = infinite_sample_li(c.L, mk(c.ref_p[0], c.ref_p[1], c.ref_p[2]), q, &wi, &pdf, &pt);
        const float r[10] = {wi.x, wi.y, wi.z, pdf, li.c[0], li.c[1], li.c[2], pt.x, pt.y, pt.z};
        for (int k = 0; k < 10; ++k) f[k] = r[k];
        break;
    }
    case DM_T_PDF: f[0] = infinite_pdf_li(c.L, mk(q[0], q[1], q[2])); break;
    case DM_T_LE: {
        const Spec v = infinite_le(c.L, mk(q[0], q[1], q[2]));
        f[0] = v.c[0], f[1] = v.c[1], f[2] = v.c[2];
        break;
    }
    case DM_T_DIFF: {
        Isect is;
        memset(&is, 0, sizeof(is));
        is.p = mk(q[0], q[1], q[2]);
        is.n = mk(q[3], q[4], q[5]);
        TexGeom g;
        memset(&g, 0, sizeof(g));
        g.dpdu = mk(q[6], q[7], q[8]);
        g.dpdv = mk(q[9], q[10], q[11]);
        const V3 r[4] = {mk(q[12], q[13], q[14]), mk(q[15], q[16], q[17]), mk(q[18], q[19], q[20]), mk(q[21], q[22], q[23])};
        compute_differentials(is, true, r, &g);
        f[0] = g.dudx, f[1] = g.dvdx, f[2] = g.dudy, f[3] = g.dvdy;
        break;
    }
    case DM_T_ROUGH: f[0] = roughness_to_alpha(q[0]); break;
    }
    for (int k = 0; k < nout; ++k) o[k] = float_as_uint(f[k]);
}

__global__ void k_tex(TexCtx c, int fam, int in, int out, const float *q, uint64_t n, uint32_t *o) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    tex_eval(c, fam, q + i * in, out, o + i * out);
}

// MIPMap::EWA's bounding box at `level` (the same arithmetic as mip_ewa), in texels; 0 past the last level
static uint64_t ewa_box(const DevMipmap &M, int level, float st0, float st1, float d00, float d01, float d10, float d11) {
    if (level >= M.levels) return 0;
    const float w = (float)M.w[level], h = (float)M.h[level];
    st0 = st0 * w - 0.5f;
    st1 = st1 * h - 0.5f;
    d00 *= w;
    d01 *= h;
    d10 *= w;
    d11 *= h;
    float A = d01 * d01 + d11 * d11 + 1;
    float B = -2 * (d00 * d01 + d10 * d11);
    float C = d00 * d00 + d10 * d10 + 1;
    const float invF = 1 / (A * C - B * B * 0.25f);
    A *= invF;
    B *= invF;
    C *= invF;
    const float det = -B * B + 4 * A * C;
    const float invDet = 1 / det;
    const float uSqrt = sqrtf(det * C), vSqrt = sqrtf(A * det);
    const float e[4] = {ceilf(st0 - 2 * invDet * uSqrt), floorf(st0 + 2 * invDet * uSqrt), ceilf(st1 - 2 * invDet * vSqrt),
                        floorf(st1 + 2 * invDet * vSqrt)};
    for (float v : e)
        if (!(std::fabs(v) < DM_ST_MAX)) return UINT64_MAX;  // NaN included
    const double ns = e[1] - e[0] + 1, nt = e[3] - e[2] + 1;
    return ns > 0 && nt > 0 ? (uint64_t)(ns * nt) : 0;
}
// The texels mip_lookup scans for one EWA query: the boxes of the two levels its lod selects (MIPMap::Lookup's ellipse
// clamp and lod, mipmap.h:276-303); UINT64_MAX when st or the box leaves the range the harness accepts
static uint64_t ewa_footprint(const DevMipmap &M, const float *q) {
    const int top = M.levels - 1;
    if (!(std::fabs(q[0] * M.w[0]) < DM_ST_MAX && std::fabs(q[1] * M.h[0]) < DM_ST_MAX)) return UINT64_MAX;
    if (M.trilinear) return 4;
    float d00 = q[2], d01 = q[3], d10 = q[4], d11 = q[5];
    if (d00 * d00 + d01 * d01 < d10 * d10 + d11 * d11) {
        std::swap(d00, d10);
        std::swap(d01, d11);
    }
    const float majorLength = sqrtf(d00 * d00 + d01 * d01);
    float minorLength = sqrtf(d10 * d10 + d11 * d11);
    if (minorLength * M.max_aniso < majorLength && minorLength > 0) {
        const float scale = majorLength / (minorLength * M.max_aniso);
        d10 *= scale;
        d11 *= scale;
        minorLength *= scale;
    }
    if (minorLength == 0) return 4;
    const float lod = pt_max((float)0, top + pt_log2f(minorLength));
    if (!(lod < 1e9f)) return UINT64_MAX;
    const int ilod = (int)floorf(lod);
    const uint64_t a = ewa_box(M, ilod, q[0], q[1], d00, d01, d10, d11), b = ewa_box(M, ilod + 1, q[0], q[1], d00, d01, d10, d11);
    return a == UINT64_MAX || b == UINT64_MAX ? UINT64_MAX : std::max(a, b);
}

static DevMipmap host_mipmap(const dm_mipmap *m, std::vector<float4> *store) {
    DevMipmap M;
    memset(&M, 0, sizeof(M));
    M.levels = m->levels;
    M.wrap = m->wrap;
    M.trilinear = m->trilinear;
    M.max_aniso = m->max_aniso;
    memcpy(M.weight_lut, m->weight_lut, sizeof(M.weight_lut));
    size_t total = 0;
    for (int l = 0; l < m->levels; ++l) total += (size_t)m->w[l] * m->h[l];
    store->resize(total);
    const float *src = m->texels;
    size_t at = 0;
    for (int l = 0; l < m->levels; ++l) {
        M.w[l] = m->w[l];
        M.h[l] = m->h[l];
        M.texels[l] = store->data() + at;
        for (size_t i = 0; i < (size_t)m->w[l] * m->h[l]; ++i, src += m->channels)
            (*store)[at++] = m->channels == 3 ? make_float4(src[0], src[1], src[2], 0.f) : make_float4(src[0], src[0], src[0], 0.f);
    }
    return M;
}

static DevInfinite host_sky(const dm_sky *s, std::vector<float4> *store) {
    DevInfinite L;
    memset(&L, 0, sizeof(L));
    L.w = s->w;
    L.h = s->h;
    store->resize((size_t)s->w * s->h);
    for (size_t i = 0; i < store->size(); ++i)
        (*store)[i] = make_float4(s->texels[3 * i], s->texels[3 * i + 1], s->texels[3 * i + 2], 0.f);
    L.texels = store->data();
    memcpy(L.light_to_world, s->light_to_world, sizeof(L.light_to_world));
    memcpy(L.world_to_light, s->world_to_light, sizeof(L.world_to_light));
    L.nu = s->nu;
    L.nv = s->nv;
    L.cond_func = s->cond_func;
    L.cond_cdf = s->cond_cdf;
    L.cond_func_int = s->cond_func_int;
    L.marg_func = s->marg_func;
    L.marg_cdf = s->marg_cdf;
    L.marg_func_int = s->marg_func_int;
    L.two_world_radius = s->two_world_radius;
    return L;
}

// Copies n elements of src to a new device allocation recorded in `owned`
template <class T>
static cudaError_t upload(const T *src, size_t n, std::vector<void *> *owned, const T **dst) {
    void *d = nullptr;
    cudaError_t e = cudaMalloc(&d, std::max<size_t>(1, n) * sizeof(T));
    if (e != cudaSuccess) return e;
    owned->push_back(d);
    *dst = (const T *)d;
    return cudaMemcpy(d, src, n * sizeof(T), cudaMemcpyHostToDevice);
}

static int tex_run(int fam, const TexCtx &host, int where, const float *q, uint64_t n, const uint32_t *want, dm_report *rep,
                   uint32_t *got, std::vector<void *> *owned, const std::vector<float4> &mipStore, const std::vector<float4> &skyStore,
                   const dm_sky *sky) {
    const int in = DM_T_IN[fam], out = DM_T_OUT[fam];
    int rc = 0;
    TexCtx dev = host;
    float *dq = nullptr;
    uint32_t *dout = nullptr;
    std::vector<uint32_t> buf;
    const uint64_t chunk = std::max<uint64_t>(1, std::min<uint64_t>(CHUNK_BYTES / (4 * (in + out)), n));
    if (where == DM_ON_DEVICE) {
        // the device copy of the tables: the same values, device pointers
        if (host.M.levels > 0) {
            const float4 *base = nullptr;
            DM_CUDA(upload(mipStore.data(), mipStore.size(), owned, &base));
            for (int l = 0; l < host.M.levels; ++l) dev.M.texels[l] = base + (host.M.texels[l] - mipStore.data());
        }
        if (sky) {
            DM_CUDA(upload(skyStore.data(), skyStore.size(), owned, &dev.L.texels));
            const size_t nu = sky->nu, nv = sky->nv;
            DM_CUDA(upload(sky->cond_func, nu * nv, owned, &dev.L.cond_func));
            DM_CUDA(upload(sky->cond_cdf, (nu + 1) * nv, owned, &dev.L.cond_cdf));
            DM_CUDA(upload(sky->cond_func_int, nv, owned, &dev.L.cond_func_int));
            DM_CUDA(upload(sky->marg_func, nv, owned, &dev.L.marg_func));
            DM_CUDA(upload(sky->marg_cdf, nv + 1, owned, &dev.L.marg_cdf));
        }
        DM_CUDA(cudaMalloc(&dq, chunk * in * 4));
        DM_CUDA(cudaMalloc(&dout, chunk * out * 4));
    }
    buf.resize(chunk * out);
    for (uint64_t s = 0; s < n; s += chunk) {
        const uint64_t m = std::min(chunk, n - s);
        if (where == DM_ON_DEVICE) {
            DM_CUDA(cudaMemcpy(dq, q + s * in, m * in * 4, cudaMemcpyHostToDevice));
            k_tex<<<(unsigned)((m + 127) / 128), 128>>>(dev, fam, in, out, dq, m, dout);
            DM_CUDA(cudaGetLastError());
            DM_CUDA(cudaMemcpy(buf.data(), dout, m * out * 4, cudaMemcpyDeviceToHost));
        } else {
            uint32_t *b = buf.data();
            parallel_for(m, [=, &host](uint64_t lo, uint64_t hi) {
                for (uint64_t i = lo; i < hi; ++i) tex_eval(host, fam, q + (s + i) * in, out, b + i * out);
            });
        }
        dm_compare(buf.data(), want + s * out, m * out, 0, s * out, 1, rep);
        if (got) std::copy(buf.begin(), buf.begin() + m * out, got + s * out);
    }
done:
    if (dq) cudaFree(dq);
    if (dout) cudaFree(dout);
    return rc;
}

static int free_all(std::vector<void *> &owned, int rc) {
    for (void *p : owned) cudaFree(p);
    return rc;
}

extern "C" {

// Per EWA query (DM_T_EWA layout), the texels mip_lookup scans (the larger of its two levels' boxes); UINT64_MAX past the
// accepted |st * size| range.  Host only: tests choose their queries with it.
int dm_mip_footprint(const dm_mipmap *m, const float *q, uint64_t n, uint64_t *texels) {
    std::vector<float4> store;
    const DevMipmap M = host_mipmap(m, &store);
    parallel_for(n, [&](uint64_t lo, uint64_t hi) {
        for (uint64_t i = lo; i < hi; ++i) texels[i] = ewa_footprint(M, q + 6 * i);
    });
    return 0;
}

// MIPMap lookups (fam DM_T_EWA or DM_T_WIDTH) of n queries against want (3 words each), on the device or host-compiled.
// The report's input is (query << 2) | word; got (optional) receives the words computed.  Refuses (-2) queries whose
// EWA footprint exceeds DM_EWA_MAX_TEXELS or whose |st * size| reaches DM_ST_MAX, before anything runs.
int dm_check_mip(const dm_mipmap *m, int fam, const float *q, uint64_t n, const uint32_t *want, int where, dm_report *rep,
                 uint32_t *got) {
    if ((fam != DM_T_EWA && fam != DM_T_WIDTH) || m->levels < 1 || m->levels > B200PT_MIPMAP_MAX_LEVELS) return -1;
    TexCtx c;
    memset(&c, 0, sizeof(c));
    std::vector<float4> store;
    c.M = host_mipmap(m, &store);
    for (uint64_t i = 0; i < n; ++i) {
        const float *e = q + (uint64_t)DM_T_IN[fam] * i;
        if (!(std::fabs(e[0] * m->w[0]) < DM_ST_MAX && std::fabs(e[1] * m->h[0]) < DM_ST_MAX)) return -2;
        if (fam == DM_T_EWA && ewa_footprint(c.M, e) > DM_EWA_MAX_TEXELS) return -2;
    }
    std::vector<void *> owned;
    return free_all(owned, tex_run(fam, c, where, q, n, want, rep, got, &owned, store, {}, nullptr));
}

// InfiniteAreaLight queries (fam DM_T_SAMPLE, DM_T_PDF or DM_T_LE) against want, on the device or host-compiled; the
// report's input is query * words + word.
int dm_check_sky(const dm_sky *s, int fam, const float *q, uint64_t n, const uint32_t *want, int where, dm_report *rep,
                 uint32_t *got) {
    if ((fam != DM_T_SAMPLE && fam != DM_T_PDF && fam != DM_T_LE) || s->w < 1 || s->h < 1 || s->nu < 1 || s->nv < 1) return -1;
    TexCtx c;
    memset(&c, 0, sizeof(c));
    std::vector<float4> store;
    c.L = host_sky(s, &store);
    memcpy(c.ref_p, s->ref_p, sizeof(c.ref_p));
    std::vector<void *> owned;
    return free_all(owned, tex_run(fam, c, where, q, n, want, rep, got, &owned, {}, store, s));
}

// ComputeDifferentials (DM_T_DIFF) or RoughnessToAlpha (DM_T_ROUGH) of n queries against want, on the device or
// host-compiled; the report's input is query * words + word.
int dm_check_geom(int fam, const float *q, uint64_t n, const uint32_t *want, int where, dm_report *rep, uint32_t *got) {
    if (fam != DM_T_DIFF && fam != DM_T_ROUGH) return -1;
    TexCtx c;
    memset(&c, 0, sizeof(c));
    std::vector<void *> owned;
    return free_all(owned, tex_run(fam, c, where, q, n, want, rep, got, &owned, {}, {}, nullptr));
}

}  // extern "C"
#endif  // DM_TEXTURE
