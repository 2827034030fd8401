// tests/devmath/devmath.cu -- TEST INFRASTRUCTURE: evaluates the path's scalar math on the device, as nvcc compiles it
// for the product (same headers, same flags: csrc/nvflags.mk), and compares it bit for bit with the host's glibc (the
// calls the reference makes) or with the host-compiled build of the same headers.  Loaded by tests/test_zz_devmath_gpu.py
// (and, without a device, by tests/test_devmath.py for its host half) through ctypes.
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
