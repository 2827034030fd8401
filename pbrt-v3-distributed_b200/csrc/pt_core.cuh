// pt_core.cuh -- device arithmetic of the path: Sobol' sampler, perspective
// camera, watertight triangle test, surface reconstruction, BSDF families,
// area-light sampling.
//
// Numerics contract: every function rounds exactly like the reference's
// scalar float code (Float=float, compiled without FMA contraction), so the
// kernels are built with -fmad=false and this header never uses fast-math
// intrinsics.  Each function cites the reference lines whose operation order
// it keeps.  The header is also compilable as plain C++ so that
// tests/host_preflight.cpp can check it on the CPU against the oracle before
// GPU time is spent (that test binary is never part of libb200pt.so).
#ifndef B200PT_CORE_CUH
#define B200PT_CORE_CUH

#include "../../include/b200pt.h"
#include "pt_platform.h"
#include "pt_sincos.cuh"
#include "pt_explog.cuh"
#include "pt_sincos_dbl.cuh"

namespace B200PT_NS {

// ------------------------------------------------------------------ constants
#define PT_MACHINE_EPS 5.9604644775390625e-08f /* 2^-24, pbrt.h:195-199 */
#define PT_PI ((float)3.14159265358979323846)
#define PT_INV_PI ((float)0.31830988618379067154)
#define PT_PI_OVER2 ((float)1.57079632679489661923)
#define PT_PI_OVER4 ((float)0.78539816339744830961)
#define PT_ONE_MINUS_EPS 0x1.fffffep-1f
#define PT_SHADOW_TMAX (1.f - 0.0001f) /* 1 - ShadowEpsilon in float, interaction.h:76 */

B200_HD float pt_inf() { return uint_as_float(0x7f800000u); }
// pbrt.h:285-287
B200_HD float pt_gamma(int n) { return (n * PT_MACHINE_EPS) / (1 - n * PT_MACHINE_EPS); }
B200_HD float pt_abs(float x) { return fabsf(x); }
// std::min / std::max semantics (second argument wins only when strictly better)
B200_HD float pt_min(float a, float b) { return (b < a) ? b : a; }
B200_HD float pt_max(float a, float b) { return (a < b) ? b : a; }
B200_HD int pt_mini(int a, int b) { return (b < a) ? b : a; }
B200_HD int pt_maxi(int a, int b) { return (a < b) ? b : a; }
B200_HD bool pt_isinf(float x) { return (float_as_uint(x) & 0x7fffffffu) == 0x7f800000u; }
B200_HD bool pt_isnan(float x) { return (float_as_uint(x) & 0x7fffffffu) > 0x7f800000u; }
// pbrt.h:300-308
B200_HD float pt_clamp(float v, float lo, float hi) {
    if (v < lo)
        return lo;
    else if (v > hi)
        return hi;
    else
        return v;
}
// pbrt.h:237-261
B200_HD float next_float_up(float v) {
    if (pt_isinf(v) && v > 0.f) return v;
    if (v == -0.f) v = 0.f;
    uint32_t ui = float_as_uint(v);
    if (v >= 0)
        ++ui;
    else
        --ui;
    return uint_as_float(ui);
}
B200_HD float next_float_down(float v) {
    if (pt_isinf(v) && v < 0.f) return v;
    if (v == 0.f) v = -0.f;
    uint32_t ui = float_as_uint(v);
    if (v > 0)
        --ui;
    else
        ++ui;
    return uint_as_float(ui);
}

// -------------------------------------------------------------------- vectors
struct V3 {
    float x, y, z;
};
B200_HD V3 mk(float x, float y, float z) {
    V3 v;
    v.x = x;
    v.y = y;
    v.z = z;
    return v;
}
B200_HD float comp(const V3 &v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : v.z); }
B200_HD V3 operator+(const V3 &a, const V3 &b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
B200_HD V3 operator-(const V3 &a, const V3 &b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
B200_HD V3 operator-(const V3 &a) { return mk(-a.x, -a.y, -a.z); }
B200_HD V3 operator*(float s, const V3 &v) { return mk(s * v.x, s * v.y, s * v.z); }
B200_HD V3 operator*(const V3 &v, float s) { return mk(s * v.x, s * v.y, s * v.z); }
B200_HD float dot(const V3 &a, const V3 &b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
B200_HD float absdot(const V3 &a, const V3 &b) { return pt_abs(dot(a, b)); }
B200_HD float len2(const V3 &v) { return v.x * v.x + v.y * v.y + v.z * v.z; }
B200_HD float len(const V3 &v) { return sqrtf(len2(v)); }
// geometry.h:243-248 (division = multiplication by the rounded reciprocal)
B200_HD V3 vdiv(const V3 &v, float f) {
    float inv = 1.0f / f;
    return mk(v.x * inv, v.y * inv, v.z * inv);
}
B200_HD V3 normalize(const V3 &v) { return vdiv(v, len(v)); }
B200_HD V3 vabs(const V3 &v) { return mk(pt_abs(v.x), pt_abs(v.y), pt_abs(v.z)); }
// geometry.h:957-963: products and differences in double, one rounding to float
B200_HD V3 cross(const V3 &a, const V3 &b) {
    double ax = a.x, ay = a.y, az = a.z, bx = b.x, by = b.y, bz = b.z;
    return mk((float)((ay * bz) - (az * by)), (float)((az * bx) - (ax * bz)), (float)((ax * by) - (ay * bx)));
}
B200_HD float max3(float a, float b, float c) { return pt_max(a, pt_max(b, c)); }
// geometry.h:1020-1027
B200_HD void coordinate_system(const V3 &v1, V3 *v2, V3 *v3) {
    if (pt_abs(v1.x) > pt_abs(v1.y))
        *v2 = vdiv(mk(-v1.z, 0.f, v1.x), sqrtf(v1.x * v1.x + v1.z * v1.z));
    else
        *v2 = vdiv(mk(0.f, v1.z, -v1.y), sqrtf(v1.y * v1.y + v1.z * v1.z));
    *v3 = cross(v1, *v2);
}

// ------------------------------------------------------------------- spectrum
// B200PT_NSPEC == 3: RGBSpectrum (core/spectrum.h:429-560), the reference's default build.
// B200PT_NSPEC == 60: SampledSpectrum (spectrum.h:283-427), the reference built with `typedef SampledSpectrum Spectrum`
// (pbrt.h:124-125).  All arithmetic is per bin (CoefficientSpectrum, spectrum.h:59-280), in bin order.
#ifdef __CUDACC__
#define PT_UNROLL _Pragma("unroll")
#else
#define PT_UNROLL
#endif
#define SPEC_FOR for (int i_ = 0; i_ < B200PT_NSPEC; ++i_)
struct Spec {
    float c[B200PT_NSPEC];
};
B200_HD Spec rgb1(float v) {
    Spec s;
    PT_UNROLL
    SPEC_FOR s.c[i_] = v;
    return s;
}
#if B200PT_NSPEC == 3
B200_HD Spec rgb(float r, float g, float b) {
    Spec c;
    c.c[0] = r;
    c.c[1] = g;
    c.c[2] = b;
    return c;
}
#endif
// spectrum stored contiguously (a descriptor's Spec triple, or one row of a 60-bin table)
B200_HD Spec rgbp(const float *p) {
    Spec s;
    PT_UNROLL
    SPEC_FOR s.c[i_] = p[i_];
    return s;
}
#define SPEC_BINOP(op)                                          \
    B200_HD Spec operator op(const Spec &a, const Spec &b) {    \
        Spec r;                                                 \
        PT_UNROLL SPEC_FOR r.c[i_] = a.c[i_] op b.c[i_]; \
        return r;                                               \
    }
SPEC_BINOP(+)
SPEC_BINOP(-)
SPEC_BINOP(*)
SPEC_BINOP(/)
#undef SPEC_BINOP
B200_HD Spec operator*(const Spec &a, float s) {
    Spec r;
    PT_UNROLL
    SPEC_FOR r.c[i_] = a.c[i_] * s;
    return r;
}
B200_HD Spec operator*(float s, const Spec &a) {
    Spec r;
    PT_UNROLL
    SPEC_FOR r.c[i_] = a.c[i_] * s;
    return r;
}
B200_HD Spec operator/(const Spec &a, float s) {  // spectrum.h:181-188
    Spec r;
    PT_UNROLL
    SPEC_FOR r.c[i_] = a.c[i_] / s;
    return r;
}
B200_HD Spec rgb_sqrt(const Spec &a) {
    Spec r;
    PT_UNROLL
    SPEC_FOR r.c[i_] = sqrtf(a.c[i_]);
    return r;
}
B200_HD bool is_black(const Spec &a) {
    bool black = true;
    PT_UNROLL
    SPEC_FOR black = black && (a.c[i_] == 0.f);
    return black;
}
B200_HD float max_comp(const Spec &a) {
    float m = a.c[0];
    PT_UNROLL
    for (int i = 1; i < B200PT_NSPEC; ++i) m = pt_max(m, a.c[i]);
    return m;
}
B200_HD bool has_nans(const Spec &a) {
    bool nan = false;
    PT_UNROLL
    SPEC_FOR nan = nan || pt_isnan(a.c[i_]);
    return nan;
}
#if B200PT_NSPEC == 3
// spectrum.h:462-465
B200_HD float lum(const Spec &a) { return 0.212671f * a.c[0] + 0.715160f * a.c[1] + 0.072169f * a.c[2]; }
#else
// SampledSpectrum::X / Y / Z (spectrum.cpp:80-100: the CIE curves averaged over the 60 bins), data of the host's
// reference build, set once per context (b200pt_scene_desc::cie_xyz).
#ifdef __CUDACC__
__constant__ float c_cie_xyz[3][B200PT_NSPEC];
#define PT_CIE_TABLE c_cie_xyz
#else
static float h_cie_xyz[3][B200PT_NSPEC];
#define PT_CIE_TABLE h_cie_xyz
#endif
#define PT_CIE(k, i) PT_CIE_TABLE[k][i]
// CIE_Y_integral = 106.856895 and sampledLambdaStart / End = 400 / 700 (spectrum.h:49-53)
#define PT_SPECTRAL_SCALE (float(700 - 400) / float(106.856895f * B200PT_NSPEC))
// spectrum.h:393-398.  Unlike ToXYZ (which multiplies by the precomputed quotient, spectrum.h:388-391) y() multiplies
// by the wavelength range first and divides afterwards -- the two round differently.
B200_HD float lum(const Spec &a) {
    float yy = 0.f;
    SPEC_FOR yy += PT_CIE(1, i_) * a.c[i_];
    return yy * float(700 - 400) / float(106.856895f * B200PT_NSPEC);
}
#endif

// ---------------------------------------------------------------------- Sobol'
struct SamplerParams {          // samplers/sobol.h:45-69
    int spp;
    int sb[4];                  // sample bounds x0 y0 x1 y1
    int resolution, log2res;
    int n_dims;
    const uint32_t *mat32;      // [n_dims][52]
    const uint32_t *table;      // device only: [n_dims][5][256] XOR of the columns selected by one index byte
    uint64_t vdc[52];
    uint64_t vdc_inv[52];
    // HaltonSampler (samplers/halton.h:60-70); type selects the sequence
    int type;                   // B200PT_SAMPLER_SOBOL / B200PT_SAMPLER_HALTON
    int base_scale[2], base_exp[2], sample_stride, mult_inverse[2];
    const uint16_t *perms;      // radicalInversePermutations
    const uint32_t *primes;     // [n_dims] Primes[d]
    const uint32_t *prime_sums; // [n_dims] PrimeSums[d]
};

// core/lowdiscrepancy.h:229-249
B200_HD uint64_t sobol_interval_to_index(const SamplerParams &sp, uint64_t frame, int px, int py) {
    const uint32_t m = (uint32_t)sp.log2res;
    if (m == 0) return 0;
    const uint32_t m2 = m << 1;
    uint64_t index = frame << m2;
    uint64_t delta = 0;
    for (int c = 0; frame; frame >>= 1, ++c)
        if (frame & 1) delta ^= sp.vdc[c];
    uint64_t b = (((uint64_t)((uint32_t)px) << m) | ((uint32_t)py)) ^ delta;
    for (int c = 0; b; b >>= 1, ++c)
        if (b & 1) index ^= sp.vdc_inv[c];
    return index;
}
// core/lowdiscrepancy.h:259-274 (+ sobol.cpp:47-59 for the two pixel dimensions)
B200_HD float sobol_sample(const SamplerParams &sp, uint64_t a, int dim, int px, int py) {
    uint32_t v = 0;
    const uint32_t *m = sp.mat32 + dim * 52;
#ifdef __CUDA_ARCH__
    // the XOR over the index bits is linear: combine five byte-indexed partial results (40 index bits)
    // instead of walking the bits one by one; any higher bits fall through to the bit loop below
    if (sp.table) {
        const uint32_t *t = sp.table + (size_t)dim * (5 * 256);
        const uint32_t lo = (uint32_t)a, hi = (uint32_t)(a >> 32);
        v = __ldg(t + (lo & 0xffu)) ^ __ldg(t + 256 + ((lo >> 8) & 0xffu)) ^ __ldg(t + 512 + ((lo >> 16) & 0xffu)) ^
            __ldg(t + 768 + (lo >> 24));
        if (hi) v ^= __ldg(t + 1024 + (hi & 0xffu));
        a >>= 40;
        m += 40;
    }
#endif
    for (; a != 0; a >>= 1, ++m)
        if (a & 1) v ^= *m;
    float s = pt_min((float)v * 0x1p-32f, PT_ONE_MINUS_EPS);
    if (dim == 0 || dim == 1) {
        s = s * (float)sp.resolution + (float)sp.sb[dim];
        s = pt_clamp(s - (float)(dim == 0 ? px : py), 0.f, PT_ONE_MINUS_EPS);
    }
    return s;
}

// ---------------------------------------------------------------------- Halton
// halton.cpp:95-116.  px, py are absolute pixel coordinates (currentPixel).
B200_HD uint64_t halton_index_for_sample(const SamplerParams &sp, uint64_t sampleNum, int px, int py) {
    int64_t offset = 0;
    if (sp.sample_stride > 1) {
        int pm[2] = {px % 128, py % 128};  // Mod(): non-negative remainder
        if (pm[0] < 0) pm[0] += 128;
        if (pm[1] < 0) pm[1] += 128;
        for (int i = 0; i < 2; ++i) {
            const uint32_t base = i == 0 ? 2u : 3u;
            uint32_t inverse = (uint32_t)pm[i];
            uint64_t dimOffset = 0;  // InverseRadicalInverse<base>, lowdiscrepancy.h:82-91
            for (int k = 0; k < sp.base_exp[i]; ++k) {
                const uint32_t digit = inverse % base;
                inverse /= base;
                dimOffset = dimOffset * base + digit;
            }
            offset += (int64_t)(dimOffset * (uint64_t)(sp.sample_stride / sp.base_scale[i]) * (uint64_t)sp.mult_inverse[i]);
        }
        offset %= sp.sample_stride;
    }
    return (uint64_t)(offset + (int64_t)sampleNum * sp.sample_stride);
}
// lowdiscrepancy.cpp:389-424: digits of `a` in `base`, reversed (optionally through a permutation);
// integer arithmetic is exact, so a run-time base gives the template's results.  32-bit division
// while the remaining value fits.
B200_HD float halton_radical_inverse(uint32_t base, const uint16_t *perm, uint64_t a) {
    const float invBase = 1.f / (float)base;
    uint64_t reversedDigits = 0;
    float invBaseN = 1.f;
    while (a >> 32) {
        const uint64_t next = a / base;
        const uint32_t digit = (uint32_t)(a - next * base);
        reversedDigits = reversedDigits * base + (perm ? (uint32_t)perm[digit] : digit);
        invBaseN *= invBase;
        a = next;
    }
    uint32_t a32 = (uint32_t)a;
    while (a32) {
        const uint32_t next = a32 / base;
        const uint32_t digit = a32 - next * base;
        reversedDigits = reversedDigits * base + (perm ? (uint32_t)perm[digit] : digit);
        invBaseN *= invBase;
        a32 = next;
    }
    if (!perm) return pt_min((float)reversedDigits * invBaseN, PT_ONE_MINUS_EPS);
    return pt_min(invBaseN * ((float)reversedDigits + invBase * (float)perm[0] / (1.f - invBase)), PT_ONE_MINUS_EPS);
}
// halton.cpp:118-127
B200_HD float halton_sample(const SamplerParams &sp, uint64_t index, int dim) {
    if (dim == 0) {  // RadicalInverse(0, a) = ReverseBits64(a) * 0x1p-64 in double (lowdiscrepancy.cpp:430-435)
        const uint64_t a = index >> sp.base_exp[0];
#ifdef __CUDA_ARCH__
        const uint64_t r = ((uint64_t)__brev((uint32_t)a) << 32) | (uint64_t)__brev((uint32_t)(a >> 32));
#else
        uint64_t r = 0;
        for (int i = 0; i < 64; ++i) r |= ((a >> i) & 1ull) << (63 - i);
#endif
        return (float)((double)r * 0x1p-64);
    }
    if (dim == 1) return halton_radical_inverse(3u, nullptr, index / (uint64_t)sp.base_scale[1]);
    return halton_radical_inverse(sp.primes[dim], sp.perms + sp.prime_sums[dim], index);
}

// Both sequences behind the GlobalSampler interface.
B200_HD uint64_t sampler_index(const SamplerParams &sp, uint64_t sampleNum, int px, int py) {
    if (sp.type == 1) return halton_index_for_sample(sp, sampleNum, px, py);
    return sobol_interval_to_index(sp, sampleNum, px - sp.sb[0], py - sp.sb[1]);  // sobol.cpp:42-45
}
B200_HD float sampler_sample(const SamplerParams &sp, uint64_t index, int dim, int px, int py) {
    if (sp.type == 1) return halton_sample(sp, index, dim);
    return sobol_sample(sp, index, dim, px, py);
}

// GlobalSampler stream state of one path (sampler.cpp:136-195): the sequence
// index of (pixel, sample) and the dimension cursor.
struct SobolStream {
    uint64_t index;
    int dim;
    int px, py;
};
B200_HD float get1d(const SamplerParams &sp, SobolStream &s) {
    float v = sampler_sample(sp, s.index, s.dim, s.px, s.py);
    s.dim += 1;
    return v;
}
B200_HD void get2d(const SamplerParams &sp, SobolStream &s, float u[2]) {
    u[0] = sampler_sample(sp, s.index, s.dim, s.px, s.py);
    u[1] = sampler_sample(sp, s.index, s.dim + 1, s.px, s.py);
    s.dim += 2;
}

// --------------------------------------------------------------------- camera
struct CameraParams {
    float r2c[16];
    float c2w[16];
    float lens_radius, focal_distance;
};
// core/transform.h:221-233
B200_HD V3 xform_point(const float *m, const V3 &p) {
    float x = p.x, y = p.y, z = p.z;
    float xp = m[0] * x + m[1] * y + m[2] * z + m[3];
    float yp = m[4] * x + m[5] * y + m[6] * z + m[7];
    float zp = m[8] * x + m[9] * y + m[10] * z + m[11];
    float wp = m[12] * x + m[13] * y + m[14] * z + m[15];
    if (wp == 1.f) return mk(xp, yp, zp);
    float inv = 1.0f / wp;
    return mk(inv * xp, inv * yp, inv * zp);
}
// core/transform.h:278-303
B200_HD V3 xform_point_err(const float *m, const V3 &p, V3 *err) {
    float x = p.x, y = p.y, z = p.z;
    float xp = m[0] * x + m[1] * y + m[2] * z + m[3];
    float yp = m[4] * x + m[5] * y + m[6] * z + m[7];
    float zp = m[8] * x + m[9] * y + m[10] * z + m[11];
    float wp = m[12] * x + m[13] * y + m[14] * z + m[15];
    float xs = (pt_abs(m[0] * x) + pt_abs(m[1] * y) + pt_abs(m[2] * z) + pt_abs(m[3]));
    float ys = (pt_abs(m[4] * x) + pt_abs(m[5] * y) + pt_abs(m[6] * z) + pt_abs(m[7]));
    float zs = (pt_abs(m[8] * x) + pt_abs(m[9] * y) + pt_abs(m[10] * z) + pt_abs(m[11]));
    *err = pt_gamma(3) * mk(xs, ys, zs);
    if (wp == 1.f) return mk(xp, yp, zp);
    float inv = 1.0f / wp;
    return mk(inv * xp, inv * yp, inv * zp);
}
// core/transform.h:235-241
B200_HD V3 xform_vector(const float *m, const V3 &v) {
    float x = v.x, y = v.y, z = v.z;
    return mk(m[0] * x + m[1] * y + m[2] * z, m[4] * x + m[5] * y + m[6] * z, m[8] * x + m[9] * y + m[10] * z);
}

// core/sampling.cpp:113-130
B200_HD void concentric_sample_disk(const float u[2], float out[2]) {
    float ux = 2.f * u[0] - 1.f, uy = 2.f * u[1] - 1.f;
    if (ux == 0.f && uy == 0.f) {
        out[0] = out[1] = 0.f;
        return;
    }
    float theta, r;
    if (pt_abs(ux) > pt_abs(uy)) {
        r = ux;
        theta = PT_PI_OVER4 * (uy / ux);
    } else {
        r = uy;
        theta = PT_PI_OVER2 - PT_PI_OVER4 * (ux / uy);
    }
    out[0] = r * pt_cosf(theta);
    out[1] = r * pt_sinf(theta);
}

// cameras/perspective.cpp:95-144 (main ray) + transform.h:251-264.  The ray
// differentials only feed image-texture filtering (interaction.cpp:103-149);
// camera_ray_differentials rebuilds them where a textured hit needs them.
B200_HD void generate_camera_ray(const CameraParams &cam, const float pFilm[2], const float uLens[2], V3 *o,
                                 V3 *d, float *tMax) {
    V3 pc = xform_point(cam.r2c, mk(pFilm[0], pFilm[1], 0.f));
    V3 ro = mk(0.f, 0.f, 0.f);
    V3 rd = normalize(pc);
    if (cam.lens_radius > 0.f) {
        float dd[2];
        concentric_sample_disk(uLens, dd);
        float lx = cam.lens_radius * dd[0], ly = cam.lens_radius * dd[1];
        float ft = cam.focal_distance / rd.z;
        V3 pFocus = ro + rd * ft;
        ro = mk(lx, ly, 0.f);
        rd = normalize(pFocus - ro);
    }
    V3 oErr;
    V3 wo = xform_point_err(cam.c2w, ro, &oErr);
    V3 wd = xform_vector(cam.c2w, rd);
    float l2 = len2(wd);
    float tm = pt_inf();
    if (l2 > 0.f) {
        float dt = dot(vabs(wd), oErr) / l2;
        wo = wo + wd * dt;
        tm -= dt;
    }
    *o = wo;
    *d = wd;
    *tMax = tm;
}

// The differentials of the camera ray generate_camera_ray makes from the same sample: cameras/perspective.cpp:117-138 in
// camera space (dxCamera / dyCamera as the constructor computes them, :55-58), CameraToWorld (transform.h:266-277, the
// offset points without error bounds) and RayDifferential::ScaleDifferentials(scale) against the world-space main ray
// (o, d) (geometry.h:946-951).  r[0..3] = rxOrigin, rxDirection, ryOrigin, ryDirection.
B200_HD void camera_ray_differentials(const CameraParams &cam, const float dxCamera[3], const float dyCamera[3], float scale,
                                      const float pFilm[2], const float uLens[2], const V3 &o, const V3 &d, V3 r[4]) {
    const V3 pc = xform_point(cam.r2c, mk(pFilm[0], pFilm[1], 0.f));
    const V3 dxc = mk(dxCamera[0], dxCamera[1], dxCamera[2]), dyc = mk(dyCamera[0], dyCamera[1], dyCamera[2]);
    V3 rxo, rxd, ryo, ryd;
    if (cam.lens_radius > 0.f) {
        float dd[2];
        concentric_sample_disk(uLens, dd);
        const float lx = cam.lens_radius * dd[0], ly = cam.lens_radius * dd[1];
        const V3 dx = normalize(pc + dxc);
        float ft = cam.focal_distance / dx.z;
        V3 pFocus = mk(0.f, 0.f, 0.f) + (ft * dx);
        rxo = mk(lx, ly, 0.f);
        rxd = normalize(pFocus - rxo);
        const V3 dy = normalize(pc + dyc);
        ft = cam.focal_distance / dy.z;
        pFocus = mk(0.f, 0.f, 0.f) + (ft * dy);
        ryo = mk(lx, ly, 0.f);
        ryd = normalize(pFocus - ryo);
    } else {
        rxo = ryo = mk(0.f, 0.f, 0.f);
        rxd = normalize(pc + dxc);
        ryd = normalize(pc + dyc);
    }
    rxo = xform_point(cam.c2w, rxo);
    ryo = xform_point(cam.c2w, ryo);
    rxd = xform_vector(cam.c2w, rxd);
    ryd = xform_vector(cam.c2w, ryd);
    r[0] = o + (rxo - o) * scale;
    r[1] = d + (rxd - d) * scale;
    r[2] = o + (ryo - o) * scale;
    r[3] = d + (ryd - d) * scale;
}

// ------------------------------------------------------------------- triangle
// Per-ray constants of the watertight test (shapes/triangle.cpp:207-219): the
// dimension permutation and the shear.  The reference recomputes them for
// every triangle; they depend on the ray only.
struct RayShear {
    int kx, ky, kz;
    float Sx, Sy, Sz;
};
B200_HD RayShear make_shear(const V3 &d) {
    RayShear s;
    V3 a = vabs(d);
    s.kz = (a.x > a.y) ? ((a.x > a.z) ? 0 : 2) : ((a.y > a.z) ? 1 : 2);  // geometry.h:998-1000
    s.kx = s.kz + 1;
    if (s.kx == 3) s.kx = 0;
    s.ky = s.kx + 1;
    if (s.ky == 3) s.ky = 0;
    float dx = comp(d, s.kx), dy = comp(d, s.ky), dz = comp(d, s.kz);
    s.Sx = -dx / dz;
    s.Sy = -dy / dz;
    s.Sz = 1.f / dz;
    return s;
}

struct TriHit {
    float t, b0, b1, b2;
};

// shapes/triangle.cpp:188-291 (== IntersectP :427-517): translate, permute,
// shear, edge functions with the fp64 fallback on an exact zero, scaled-t
// range test against ray.tMax, then the conservative t > deltaT check.
B200_HD bool triangle_test(const V3 &p0, const V3 &p1, const V3 &p2, const V3 &ro, const RayShear &sh,
                           float rayTMax, TriHit *h) {
    V3 q0 = p0 - ro, q1 = p1 - ro, q2 = p2 - ro;
    float p0x = comp(q0, sh.kx), p0y = comp(q0, sh.ky), p0z = comp(q0, sh.kz);
    float p1x = comp(q1, sh.kx), p1y = comp(q1, sh.ky), p1z = comp(q1, sh.kz);
    float p2x = comp(q2, sh.kx), p2y = comp(q2, sh.ky), p2z = comp(q2, sh.kz);
    p0x += sh.Sx * p0z;
    p0y += sh.Sy * p0z;
    p1x += sh.Sx * p1z;
    p1y += sh.Sy * p1z;
    p2x += sh.Sx * p2z;
    p2y += sh.Sy * p2z;
    float e0 = p1x * p2y - p1y * p2x;
    float e1 = p2x * p0y - p2y * p0x;
    float e2 = p0x * p1y - p0y * p1x;
    if (e0 == 0.0f || e1 == 0.0f || e2 == 0.0f) {
        double p2txp1ty = (double)p2x * (double)p1y;
        double p2typ1tx = (double)p2y * (double)p1x;
        e0 = (float)(p2typ1tx - p2txp1ty);
        double p0txp2ty = (double)p0x * (double)p2y;
        double p0typ2tx = (double)p0y * (double)p2x;
        e1 = (float)(p0typ2tx - p0txp2ty);
        double p1txp0ty = (double)p1x * (double)p0y;
        double p1typ0tx = (double)p1y * (double)p0x;
        e2 = (float)(p1typ0tx - p1txp0ty);
    }
    if ((e0 < 0 || e1 < 0 || e2 < 0) && (e0 > 0 || e1 > 0 || e2 > 0)) return false;
    float det = e0 + e1 + e2;
    if (det == 0) return false;
    p0z *= sh.Sz;
    p1z *= sh.Sz;
    p2z *= sh.Sz;
    float tScaled = e0 * p0z + e1 * p1z + e2 * p2z;
    if (det < 0 && (tScaled >= 0 || tScaled < rayTMax * det))
        return false;
    else if (det > 0 && (tScaled <= 0 || tScaled > rayTMax * det))
        return false;
    float invDet = 1 / det;
    float b0 = e0 * invDet;
    float b1 = e1 * invDet;
    float b2 = e2 * invDet;
    float t = tScaled * invDet;
    float maxZt = max3(pt_abs(p0z), pt_abs(p1z), pt_abs(p2z));
    float deltaZ = pt_gamma(3) * maxZt;
    float maxXt = max3(pt_abs(p0x), pt_abs(p1x), pt_abs(p2x));
    float maxYt = max3(pt_abs(p0y), pt_abs(p1y), pt_abs(p2y));
    float deltaX = pt_gamma(5) * (maxXt + maxZt);
    float deltaY = pt_gamma(5) * (maxYt + maxZt);
    float deltaE = 2 * (pt_gamma(2) * maxXt * maxYt + deltaY * maxXt + deltaX * maxYt);
    float maxE = max3(pt_abs(e0), pt_abs(e1), pt_abs(e2));
    float deltaT = 3 * (pt_gamma(3) * maxE * maxZt + deltaE * maxZt + deltaZ * maxE) * pt_abs(invDet);
    if (t <= deltaT) return false;
    h->t = t;
    h->b0 = b0;
    h->b1 = b1;
    h->b2 = b2;
    return true;
}

// shapes/triangle.cpp:293-318.  false = degenerate triangle (the reference then
// reports no intersection at all).
// Per-vertex shading data of a triangle: TriangleMesh::n and ::uv gathered through the index buffer.
struct TriShading {
    int has_n;
    V3 n0, n1, n2;
    float uv[6];  // (u,v) of the three vertices; Triangle::GetUVs defaults (0,0),(1,0),(1,1) without mesh uvs
};
B200_HD void default_shading(TriShading *t) {
    t->has_n = 0;
    t->uv[0] = 0.f;
    t->uv[1] = 0.f;
    t->uv[2] = 1.f;
    t->uv[3] = 0.f;
    t->uv[4] = 1.f;
    t->uv[5] = 1.f;
}
B200_HD bool triangle_partials(const V3 &p0, const V3 &p1, const V3 &p2, const float *uv, V3 *dpdu, V3 *dpdv) {
    const float uv0x = uv[0], uv0y = uv[1], uv1x = uv[2], uv1y = uv[3], uv2x = uv[4], uv2y = uv[5];
    float duv02x = uv0x - uv2x, duv02y = uv0y - uv2y;
    float duv12x = uv1x - uv2x, duv12y = uv1y - uv2y;
    V3 dp02 = p0 - p2, dp12 = p1 - p2;
    float determinant = duv02x * duv12y - duv02y * duv12x;
    bool degenerateUV = pt_abs(determinant) < 1e-8f;
    if (!degenerateUV) {
        float invdet = 1 / determinant;
        *dpdu = (duv12y * dp02 - duv02y * dp12) * invdet;
        *dpdv = (-duv12x * dp02 + duv02x * dp12) * invdet;
    }
    if (degenerateUV || len2(cross(*dpdu, *dpdv)) == 0) {
        V3 ng = cross(p2 - p0, p1 - p0);
        if (len2(ng) == 0) return false;
        coordinate_system(normalize(ng), dpdu, dpdv);
    }
    return true;
}

// shapes/triangle.cpp:575-581
B200_HD float triangle_area(const V3 &p0, const V3 &p1, const V3 &p2) {
    return (float)(0.5 * (double)len(cross(p1 - p0, p2 - p0)));
}

// SurfaceInteraction of a triangle hit (meshes without per-vertex tangents):
// triangle.cpp:293-425 and interaction.cpp:44-92.
struct Isect {
    V3 p, pError, n, wo;  // n = geometric normal after orientation
    V3 ns;                // shading.n
    V3 sdpdu;             // shading.dpdu
};
// What texture lookups need of a surface hit besides Isect: the geometric SurfaceInteraction::dpdu / dpdv and uv (world
// space, like the hit) and the screen-space uv derivatives ComputeDifferentials leaves
struct TexGeom {
    V3 dpdu, dpdv;
    float u, v;
    float dudx, dvdx, dudy, dvdy;
};
// SurfaceInteraction::ComputeDifferentials (interaction.cpp:103-149) for a ray with differentials r[0..3] = rxOrigin,
// rxDirection, ryOrigin, ryDirection; has_diff == false (or a failed plane intersection) zeroes the derivatives
B200_HD void compute_differentials(const Isect &is, bool has_diff, const V3 r[4], TexGeom *g) {
    g->dudx = g->dvdx = g->dudy = g->dvdy = 0.f;
    if (!has_diff) return;
    const V3 n = is.n, p = is.p;
    const float d = dot(n, p);
    const float tx = -(dot(n, r[0]) - d) / dot(n, r[1]);
    if (pt_isinf(tx) || tx != tx) return;
    const V3 px = r[0] + tx * r[1];
    const float ty = -(dot(n, r[2]) - d) / dot(n, r[3]);
    if (pt_isinf(ty) || ty != ty) return;
    const V3 py = r[2] + ty * r[3];
    int d0, d1;
    if (pt_abs(n.x) > pt_abs(n.y) && pt_abs(n.x) > pt_abs(n.z)) {
        d0 = 1;
        d1 = 2;
    } else if (pt_abs(n.y) > pt_abs(n.z)) {
        d0 = 0;
        d1 = 2;
    } else {
        d0 = 0;
        d1 = 1;
    }
    const float A00 = comp(g->dpdu, d0), A01 = comp(g->dpdv, d0), A10 = comp(g->dpdu, d1), A11 = comp(g->dpdv, d1);
    // SolveLinearSystem2x2 (transform.cpp:41-49); a failed solve leaves its pair at 0
    auto solve = [&](float b0, float b1, float *x0, float *x1) {
        const float det = A00 * A11 - A01 * A10;
        if (pt_abs(det) < 1e-10f) return;
        const float y0 = (A11 * b0 - A01 * b1) / det;
        const float y1 = (A00 * b1 - A10 * b0) / det;
        if (y0 != y0 || y1 != y1) return;
        *x0 = y0;
        *x1 = y1;
    };
    solve(comp(px, d0) - comp(p, d0), comp(px, d1) - comp(p, d1), &g->dudx, &g->dvdx);
    solve(comp(py, d0) - comp(p, d0), comp(py, d1) - comp(p, d1), &g->dudy, &g->dvdy);
}

B200_HD void fill_isect(const V3 &p0, const V3 &p1, const V3 &p2, bool flip, const TriShading &sh, const TriHit &h,
                        const V3 &rayD, Isect *is) {
    V3 dpdu, dpdv;
    triangle_partials(p0, p1, p2, sh.uv, &dpdu, &dpdv);
    float xs = (pt_abs(h.b0 * p0.x) + pt_abs(h.b1 * p1.x) + pt_abs(h.b2 * p2.x));
    float ys = (pt_abs(h.b0 * p0.y) + pt_abs(h.b1 * p1.y) + pt_abs(h.b2 * p2.y));
    float zs = (pt_abs(h.b0 * p0.z) + pt_abs(h.b1 * p1.z) + pt_abs(h.b2 * p2.z));
    is->pError = pt_gamma(7) * mk(xs, ys, zs);
    is->p = h.b0 * p0 + h.b1 * p1 + h.b2 * p2;
    is->wo = normalize(-rayD);
    V3 n = normalize(cross(p0 - p2, p1 - p2));  // triangle.cpp:341
    is->ns = n;
    is->sdpdu = dpdu;
    if (sh.has_n) {
        // triangle.cpp:342-413 + SetShadingGeometry(ss, ts, ..., true), interaction.cpp:73-92
        V3 ns = (h.b0 * sh.n0 + h.b1 * sh.n1 + h.b2 * sh.n2);
        if (len2(ns) > 0)
            ns = normalize(ns);
        else
            ns = n;
        V3 ss = normalize(dpdu);
        V3 ts = cross(ss, ns);
        if (len2(ts) > 0.f) {
            ts = normalize(ts);
            ss = cross(ts, ns);
        } else
            coordinate_system(ns, &ss, &ts);
        V3 sn = normalize(cross(ss, ts));
        if (flip) sn = -sn;
        n = (dot(n, sn) < 0.f) ? -n : n;   // Faceforward(n, shading.n)
        is->ns = sn;
        is->sdpdu = ss;
        n = (dot(n, is->ns) < 0.f) ? -n : n;  // triangle.cpp:418-419
    } else if (flip) {
        n = -n;  // triangle.cpp:420-421
        is->ns = n;
    }
    is->n = n;
}

// The triangle's SurfaceInteraction::dpdu / dpdv and uv (triangle.cpp:293-318, :329-330)
B200_HD void triangle_tex_geom(const V3 &p0, const V3 &p1, const V3 &p2, const TriShading &sh, const TriHit &h, TexGeom *g) {
    triangle_partials(p0, p1, p2, sh.uv, &g->dpdu, &g->dpdv);
    g->u = h.b0 * sh.uv[0] + h.b1 * sh.uv[2] + h.b2 * sh.uv[4];
    g->v = h.b0 * sh.uv[1] + h.b1 * sh.uv[3] + h.b2 * sh.uv[5];
}

// core/geometry.h:1440-1460
B200_HD V3 offset_ray_origin(const V3 &p, const V3 &pError, const V3 &n, const V3 &w) {
    float d = dot(vabs(n), pError);
    V3 offset = d * n;
    if (dot(w, n) < 0) offset = -offset;
    V3 po = p + offset;
    if (offset.x > 0)
        po.x = next_float_up(po.x);
    else if (offset.x < 0)
        po.x = next_float_down(po.x);
    if (offset.y > 0)
        po.y = next_float_up(po.y);
    else if (offset.y < 0)
        po.y = next_float_down(po.y);
    if (offset.z > 0)
        po.z = next_float_up(po.z);
    else if (offset.z < 0)
        po.z = next_float_down(po.z);
    return po;
}

// ---------------------------------------------------------------------- BSDFs
enum {
    BSDF_REFLECTION = 1,
    BSDF_TRANSMISSION = 2,
    BSDF_DIFFUSE = 4,
    BSDF_GLOSSY = 8,
    BSDF_SPECULAR = 16,
    BSDF_ALL = 31
};

B200_HD float cos_theta(const V3 &w) { return w.z; }
B200_HD float cos2_theta(const V3 &w) { return w.z * w.z; }
B200_HD float abs_cos_theta(const V3 &w) { return pt_abs(w.z); }
B200_HD float sin2_theta(const V3 &w) { return pt_max(0.f, 1.f - cos2_theta(w)); }
B200_HD float sin_theta(const V3 &w) { return sqrtf(sin2_theta(w)); }
B200_HD float tan_theta(const V3 &w) { return sin_theta(w) / cos_theta(w); }
B200_HD float tan2_theta(const V3 &w) { return sin2_theta(w) / cos2_theta(w); }
B200_HD float cos_phi(const V3 &w) {
    float st = sin_theta(w);
    return (st == 0) ? 1.f : pt_clamp(w.x / st, -1.f, 1.f);
}
B200_HD float sin_phi(const V3 &w) {
    float st = sin_theta(w);
    return (st == 0) ? 0.f : pt_clamp(w.y / st, -1.f, 1.f);
}
B200_HD float cos2_phi(const V3 &w) { return cos_phi(w) * cos_phi(w); }
B200_HD float sin2_phi(const V3 &w) { return sin_phi(w) * sin_phi(w); }
B200_HD bool same_hemisphere(const V3 &w, const V3 &wp) { return w.z * wp.z > 0; }
B200_HD V3 reflect(const V3 &wo, const V3 &n) { return -wo + 2 * dot(wo, n) * n; }  // reflection.h:97-99
// reflection.h:101-114
B200_HD bool refract(const V3 &wi, const V3 &n, float eta, V3 *wt) {
    float cosThetaI = dot(n, wi);
    float sin2ThetaI = pt_max(0.f, 1 - cosThetaI * cosThetaI);
    float sin2ThetaT = eta * eta * sin2ThetaI;
    if (sin2ThetaT >= 1) return false;
    float cosThetaT = sqrtf(1 - sin2ThetaT);
    *wt = eta * -wi + (eta * cosThetaI - cosThetaT) * n;
    return true;
}
// reflection.cpp:47-68
B200_HD float fr_dielectric(float cosThetaI, float etaI, float etaT) {
    cosThetaI = pt_clamp(cosThetaI, -1.f, 1.f);
    bool entering = cosThetaI > 0.f;
    if (!entering) {
        float t = etaI;
        etaI = etaT;
        etaT = t;
        cosThetaI = pt_abs(cosThetaI);
    }
    float sinThetaI = sqrtf(pt_max(0.f, 1 - cosThetaI * cosThetaI));
    float sinThetaT = etaI / etaT * sinThetaI;
    if (sinThetaT >= 1) return 1;
    float cosThetaT = sqrtf(pt_max(0.f, 1 - sinThetaT * sinThetaT));
    float Rparl = ((etaT * cosThetaI) - (etaI * cosThetaT)) / ((etaT * cosThetaI) + (etaI * cosThetaT));
    float Rperp = ((etaI * cosThetaI) - (etaT * cosThetaT)) / ((etaI * cosThetaI) + (etaT * cosThetaT));
    return (Rparl * Rparl + Rperp * Rperp) / 2;
}
// reflection.cpp:71-94
B200_HD Spec fr_conductor(float cosThetaI, const Spec &etai, const Spec &etat, const Spec &k) {
    cosThetaI = pt_clamp(cosThetaI, -1.f, 1.f);
    Spec eta = etat / etai;
    Spec etak = k / etai;
    float cosThetaI2 = cosThetaI * cosThetaI;
    float sinThetaI2 = (float)(1. - (double)cosThetaI2);
    Spec eta2 = eta * eta;
    Spec etak2 = etak * etak;
    Spec t0 = eta2 - etak2 - rgb1(sinThetaI2);
    Spec a2plusb2 = rgb_sqrt(t0 * t0 + 4.f * eta2 * etak2);
    Spec t1 = a2plusb2 + rgb1(cosThetaI2);
    Spec a = rgb_sqrt(0.5f * (a2plusb2 + t0));
    Spec t2 = (2.f * cosThetaI) * a;
    Spec Rs = (t1 - t2) / (t1 + t2);
    Spec t3 = cosThetaI2 * a2plusb2 + rgb1(sinThetaI2 * sinThetaI2);
    Spec t4 = t2 * sinThetaI2;
    Spec Rp = Rs * (t3 - t4) / (t3 + t4);
    return 0.5f * (Rp + Rs);
}

// TrowbridgeReitzDistribution with sampleVisibleArea = true (the materials' default)
struct TRDist {
    float ax, ay;
};
// microfacet.cpp:155-163
B200_HD float tr_D(const TRDist &d, const V3 &wh) {
    float tan2Theta = tan2_theta(wh);
    if (pt_isinf(tan2Theta)) return 0.f;
    const float cos4Theta = cos2_theta(wh) * cos2_theta(wh);
    float e = (cos2_phi(wh) / (d.ax * d.ax) + sin2_phi(wh) / (d.ay * d.ay)) * tan2Theta;
    return 1 / (PT_PI * d.ax * d.ay * cos4Theta * (1 + e) * (1 + e));
}
// microfacet.cpp:176-184
B200_HD float tr_lambda(const TRDist &d, const V3 &w) {
    float absTanTheta = pt_abs(tan_theta(w));
    if (pt_isinf(absTanTheta)) return 0.f;
    float alpha = sqrtf(cos2_phi(w) * d.ax * d.ax + sin2_phi(w) * d.ay * d.ay);
    float alpha2Tan2Theta = (alpha * absTanTheta) * (alpha * absTanTheta);
    return (-1 + sqrtf(1.f + alpha2Tan2Theta)) / 2;
}
B200_HD float tr_G1(const TRDist &d, const V3 &w) { return 1 / (1 + tr_lambda(d, w)); }            // microfacet.h:54-57
B200_HD float tr_G(const TRDist &d, const V3 &wo, const V3 &wi) { return 1 / (1 + tr_lambda(d, wo) + tr_lambda(d, wi)); }
// microfacet.cpp:338-344
B200_HD float tr_pdf(const TRDist &d, const V3 &wo, const V3 &wh) {
    return tr_D(d, wh) * tr_G1(d, wo) * absdot(wo, wh) / abs_cos_theta(wo);
}
// microfacet.cpp:238-283.  The normal-incidence branch calls the C `cos`/`sin`
// on a float (promoted to double) and multiplies in double; pt_cos / pt_sin
// (pt_sincos_dbl.cuh) round like the host's glibc, which libdevice's do not.
B200_HD_L2 void tr_sample11(float cosTheta, float U1, float U2, float *slope_x, float *slope_y) {
    if ((double)cosTheta > .9999) {
        float r = sqrtf(U1 / (1 - U1));
        float phi = (float)(6.28318530718 * (double)U2);
        *slope_x = (float)((double)r * pt_cos((double)phi));
        *slope_y = (float)((double)r * pt_sin((double)phi));
        return;
    }
    float sinTheta = sqrtf(pt_max(0.f, 1.f - cosTheta * cosTheta));
    float tanTheta = sinTheta / cosTheta;
    float a = 1 / tanTheta;
    float G1 = 2 / (1 + sqrtf(1.f + 1.f / (a * a)));
    float A = 2 * U1 / G1 - 1;
    float tmp = 1.f / (A * A - 1.f);
    if (tmp > 1e10f) tmp = 1e10f;
    float B = tanTheta;
    float D = sqrtf(pt_max(B * B * tmp * tmp - (A * A - B * B) * tmp, 0.f));
    float slope_x_1 = B * tmp - D;
    float slope_x_2 = B * tmp + D;
    *slope_x = (A < 0 || slope_x_2 > 1.f / tanTheta) ? slope_x_1 : slope_x_2;
    float S;
    if (U2 > 0.5f) {
        S = 1.f;
        U2 = 2.f * (U2 - .5f);
    } else {
        S = -1.f;
        U2 = 2.f * (.5f - U2);
    }
    float z = (U2 * (U2 * (U2 * 0.27385f - 0.73369f) + 0.46341f)) /
              (U2 * (U2 * (U2 * 0.093073f + 0.309420f) - 1.000000f) + 0.597999f);
    *slope_y = S * z * sqrtf(1.f + *slope_x * *slope_x);
}
// microfacet.cpp:285-305
B200_HD V3 tr_sample(const V3 &wi, float ax, float ay, float U1, float U2) {
    V3 ws = normalize(mk(ax * wi.x, ay * wi.y, wi.z));
    float sx, sy;
    tr_sample11(cos_theta(ws), U1, U2, &sx, &sy);
    float tmp = cos_phi(ws) * sx - sin_phi(ws) * sy;
    sy = sin_phi(ws) * sx + cos_phi(ws) * sy;
    sx = tmp;
    sx = ax * sx;
    sy = ay * sy;
    return normalize(mk(-sx, -sy, 1.f));
}
// microfacet.cpp:307-336 (visible-area branch)
B200_HD V3 tr_sample_wh(const TRDist &d, const V3 &wo, const float u[2]) {
    bool flip = wo.z < 0;
    V3 wh = tr_sample(flip ? -wo : wo, d.ax, d.ay, u[0], u[1]);
    if (flip) wh = -wh;
    return wh;
}
// sampling.h:159-163
B200_HD V3 cosine_sample_hemisphere(const float u[2]) {
    float d[2];
    concentric_sample_disk(u, d);
    float z = sqrtf(pt_max(0.f, 1 - d[0] * d[0] - d[1] * d[1]));
    return mk(d[0], d[1], z);
}

// One BxDF lobe.  kind: 0 Lambertian, 1 MicrofacetReflection (TR), 2 FresnelSpecular, 3 OrenNayar,
// 4 MicrofacetTransmission (TR)
enum { BX_LAMBERT = 0, BX_MICROFACET = 1, BX_FRESNEL_SPECULAR = 2, BX_OREN_NAYAR = 3, BX_MICROFACET_TRANS = 4,
       BX_SPECULAR_REFLECTION = 5 };
// The lobe kinds a material family can produce (make_bsdf): the per-family shading kernels pass this mask down as a
// template argument, so each carries only its own BxDFs' code (the lobes themselves stay run-time data).  ncu showed
// the shading kernels' warps waiting for instruction fetches; the plastic kernel does not need the conductor's
// Fresnel term, rough-glass transmission or Oren-Nayar.
#define KM(k) (1 << (k))
#define KM_DIEL 0x100  // microfacet reflection with FresnelDielectric
#define KM_COND 0x200  // ... with FresnelConductor
#define KM_ALL 0x3ff
#define KM_CONST 0x400  // (lazy spectra) the constant recipe LT_CONST: only the medium vertex asks for it
B200_HD constexpr int mat_kinds(int material) {
    return material == 0   ? (KM(BX_LAMBERT) | KM(BX_OREN_NAYAR))                  // B200PT_MAT_MATTE
           : material == 1 ? (KM(BX_LAMBERT) | KM(BX_MICROFACET) | KM_DIEL)        // B200PT_MAT_PLASTIC
           : material == 2 ? (KM(BX_MICROFACET) | KM_COND)                         // B200PT_MAT_METAL
           : material == 3 ? (KM(BX_MICROFACET) | KM_DIEL | KM(BX_MICROFACET_TRANS) | KM(BX_FRESNEL_SPECULAR) |
                              KM(BX_SPECULAR_REFLECTION))                          // B200PT_MAT_GLASS (smooth, rough, mirror)
                           : KM_ALL;
}
// A lobe's spectra are rows of the material table (or the constant 1).  The RGBSpectrum build keeps them by value in
// registers; the SampledSpectrum build keeps a pointer to the row -- 60 floats per spectrum copied into every thread's
// Bsdf were a third of k_shade's 6.4 KB local-memory frame, and the rows are shared by all threads (L1 hits).
#if B200PT_NSPEC == 3
typedef Spec SpecRef;
B200_HD SpecRef sref(const float *p) { return rgbp(p); }
B200_HD SpecRef sref_one() { return rgb1(1.f); }
B200_HD const Spec &sval(const SpecRef &r) { return r; }
#else
struct SpecRef {
    const float *p;  // nullptr: the constant spectrum 1
};
B200_HD SpecRef sref(const float *p) {
    SpecRef r;
    r.p = p;
    return r;
}
B200_HD SpecRef sref_one() { return sref(nullptr); }
B200_HD Spec sval(const SpecRef &r) { return r.p ? rgbp(r.p) : rgb1(1.f); }
#endif
struct Lobe {
    int kind, type;
    SpecRef R, T;
    TRDist dist;
    int conductor;      // Fresnel of the microfacet lobe: 0 dielectric(etaI, etaT), 1 conductor(1, cEta, cK)
    float frEtaI, frEtaT;
    SpecRef cEta, cK;
    float etaA, etaB;   // FresnelSpecular, MicrofacetTransmission
    float onA, onB;     // OrenNayar
};
B200_HD bool lobe_matches(const Lobe &l, int flags) { return (l.type & flags) == l.type; }
template <int KINDS = KM_ALL>
B200_HD Spec lobe_fresnel(const Lobe &l, float cosThetaI) {
    if (!(KINDS & KM_COND) || ((KINDS & KM_DIEL) && !l.conductor))
        return rgb1(fr_dielectric(cosThetaI, l.frEtaI, l.frEtaT));  // reflection.cpp:128-130
    return fr_conductor(pt_abs(cosThetaI), rgb1(1.f), sval(l.cEta), sval(l.cK));               // reflection.cpp:117-119
}
template <int KINDS = KM_ALL>
B200_HD_L2 Spec lobe_f(const Lobe &l, const V3 &wo, const V3 &wi) {
    if ((KINDS & KM(BX_LAMBERT)) && l.kind == BX_LAMBERT) return sval(l.R) * PT_INV_PI;  // reflection.cpp:178-180
    if ((KINDS & KM(BX_MICROFACET)) && l.kind == BX_MICROFACET) {                     // reflection.cpp:226-236
        float cosThetaO = abs_cos_theta(wo), cosThetaI = abs_cos_theta(wi);
        V3 wh = wi + wo;
        if (cosThetaI == 0 || cosThetaO == 0) return rgb1(0.f);
        if (wh.x == 0 && wh.y == 0 && wh.z == 0) return rgb1(0.f);
        wh = normalize(wh);
        Spec F = lobe_fresnel<KINDS>(l, dot(wi, wh));
        return sval(l.R) * tr_D(l.dist, wh) * tr_G(l.dist, wo, wi) * F / (4 * cosThetaI * cosThetaO);
    }
    if ((KINDS & KM(BX_OREN_NAYAR)) && l.kind == BX_OREN_NAYAR) {  // reflection.cpp:197-219
        float sinThetaI = sin_theta(wi);
        float sinThetaO = sin_theta(wo);
        float maxCos = 0;
        if ((double)sinThetaI > 1e-4 && (double)sinThetaO > 1e-4) {
            float sinPhiI = sin_phi(wi), cosPhiI = cos_phi(wi);
            float sinPhiO = sin_phi(wo), cosPhiO = cos_phi(wo);
            float dCos = cosPhiI * cosPhiO + sinPhiI * sinPhiO;
            maxCos = pt_max(0.f, dCos);
        }
        float sinAlpha, tanBeta;
        if (abs_cos_theta(wi) > abs_cos_theta(wo)) {
            sinAlpha = sinThetaO;
            tanBeta = sinThetaI / abs_cos_theta(wi);
        } else {
            sinAlpha = sinThetaI;
            tanBeta = sinThetaO / abs_cos_theta(wo);
        }
        return sval(l.R) * PT_INV_PI * (l.onA + l.onB * maxCos * sinAlpha * tanBeta);
    }
    if ((KINDS & KM(BX_MICROFACET_TRANS)) && l.kind == BX_MICROFACET_TRANS) {  // reflection.cpp:244-266 (TransportMode::Radiance)
        if (same_hemisphere(wo, wi)) return rgb1(0.f);
        float cosThetaO = cos_theta(wo);
        float cosThetaI = cos_theta(wi);
        if (cosThetaI == 0 || cosThetaO == 0) return rgb1(0.f);
        float eta = cos_theta(wo) > 0 ? (l.etaB / l.etaA) : (l.etaA / l.etaB);
        V3 wh = normalize(wo + wi * eta);
        if (wh.z < 0) wh = -wh;
        Spec F = rgb1(fr_dielectric(dot(wo, wh), l.etaA, l.etaB));
        float sqrtDenom = dot(wo, wh) + eta * dot(wi, wh);
        float factor = 1 / eta;
        return (rgb1(1.f) - F) * sval(l.T) *
               pt_abs(tr_D(l.dist, wh) * tr_G(l.dist, wo, wi) * eta * eta * absdot(wi, wh) * absdot(wo, wh) * factor *
                      factor / (cosThetaI * cosThetaO * sqrtDenom * sqrtDenom));
    }
    return rgb1(0.f);  // FresnelSpecular::f, reflection.h:363-365
}
template <int KINDS = KM_ALL>
B200_HD_L2 float lobe_pdf(const Lobe &l, const V3 &wo, const V3 &wi) {
    if ((KINDS & (KM(BX_LAMBERT) | KM(BX_OREN_NAYAR))) && (l.kind == BX_LAMBERT || l.kind == BX_OREN_NAYAR))
        return same_hemisphere(wo, wi) ? abs_cos_theta(wi) * PT_INV_PI : 0.f;  // reflection.cpp:387-389
    if ((KINDS & KM(BX_MICROFACET_TRANS)) && l.kind == BX_MICROFACET_TRANS) {  // reflection.cpp:436-448
        if (same_hemisphere(wo, wi)) return 0.f;
        float eta = cos_theta(wo) > 0 ? (l.etaB / l.etaA) : (l.etaA / l.etaB);
        V3 wh = normalize(wo + wi * eta);
        float sqrtDenom = dot(wo, wh) + eta * dot(wi, wh);
        float dwh_dwi = pt_abs((eta * eta * dot(wi, wh)) / (sqrtDenom * sqrtDenom));
        return tr_pdf(l.dist, wo, wh) * dwh_dwi;
    }
    if ((KINDS & KM(BX_MICROFACET)) && l.kind == BX_MICROFACET) {                                    // reflection.cpp:419-423
        if (!same_hemisphere(wo, wi)) return 0.f;
        V3 wh = normalize(wo + wi);
        return tr_pdf(l.dist, wo, wh) / (4 * dot(wo, wh));
    }
    return 0.f;
}
// BxDF::Sample_f; *pdf is written only where the reference writes it.
template <int KINDS = KM_ALL>
B200_HD_L2 Spec lobe_sample_f(const Lobe &l, const V3 &wo, V3 *wi, const float u[2], float *pdf, int *sampledType) {
    if ((KINDS & KM(BX_MICROFACET_TRANS)) && l.kind == BX_MICROFACET_TRANS) {  // reflection.cpp:425-434
        if (wo.z == 0) return rgb1(0.f);
        V3 wh = tr_sample_wh(l.dist, wo, u);
        float eta = cos_theta(wo) > 0 ? (l.etaA / l.etaB) : (l.etaB / l.etaA);
        if (!refract(wo, wh, eta, wi)) return rgb1(0.f);
        *pdf = lobe_pdf<KINDS>(l, wo, *wi);
        return lobe_f<KINDS>(l, wo, *wi);
    }
    if ((KINDS & (KM(BX_LAMBERT) | KM(BX_OREN_NAYAR))) && (l.kind == BX_LAMBERT || l.kind == BX_OREN_NAYAR)) {  // BxDF::Sample_f, reflection.cpp:378-385
        *wi = cosine_sample_hemisphere(u);
        if (wo.z < 0) wi->z *= -1;
        *pdf = lobe_pdf<KINDS>(l, wo, *wi);
        return lobe_f<KINDS>(l, wo, *wi);
    }
    if ((KINDS & KM(BX_MICROFACET)) && l.kind == BX_MICROFACET) {  // reflection.cpp:405-417
        if (wo.z == 0) return rgb1(0.f);
        V3 wh = tr_sample_wh(l.dist, wo, u);
        *wi = reflect(wo, wh);
        if (!same_hemisphere(wo, *wi)) return rgb1(0.f);
        *pdf = tr_pdf(l.dist, wo, wh) / (4 * dot(wo, wh));
        return lobe_f<KINDS>(l, wo, *wi);
    }
    if ((KINDS & KM(BX_SPECULAR_REFLECTION)) && l.kind == BX_SPECULAR_REFLECTION) {  // reflection.cpp:136-143 with FresnelNoOp (mirror.cpp:45-56)
        *wi = mk(-wo.x, -wo.y, wo.z);
        *pdf = 1.f;
        return rgb1(1.f) * sval(l.R) / abs_cos_theta(*wi);
    }
    if (!(KINDS & KM(BX_FRESNEL_SPECULAR))) return rgb1(0.f);  // (no such lobe in this family)
    // FresnelSpecular::Sample_f, reflection.cpp:477-511 (TransportMode::Radiance)
    float F = fr_dielectric(cos_theta(wo), l.etaA, l.etaB);
    if (u[0] < F) {
        *wi = mk(-wo.x, -wo.y, wo.z);
        *sampledType = BSDF_SPECULAR | BSDF_REFLECTION;
        *pdf = F;
        return F * sval(l.R) / abs_cos_theta(*wi);
    }
    bool entering = cos_theta(wo) > 0;
    float etaI = entering ? l.etaA : l.etaB;
    float etaT = entering ? l.etaB : l.etaA;
    V3 nn = mk(0.f, 0.f, 1.f);
    if (dot(nn, wo) < 0.f) nn = -nn;  // Faceforward, geometry.h:1213-1216
    if (!refract(wo, nn, etaI / etaT, wi)) return rgb1(0.f);
    Spec ft = sval(l.T) * (1 - F);
    ft = ft * ((etaI * etaI) / (etaT * etaT));
    *sampledType = BSDF_SPECULAR | BSDF_TRANSMISSION;
    *pdf = 1 - F;
    return ft / abs_cos_theta(*wi);
}

// BSDF (reflection.h:153-202) with at most two lobes
struct Bsdf {
    float eta;
    V3 ns, ng, ss, ts;
    int n;
    Lobe lobes[2];
};
B200_HD V3 world_to_local(const Bsdf &b, const V3 &v) { return mk(dot(v, b.ss), dot(v, b.ts), dot(v, b.ns)); }
B200_HD V3 local_to_world(const Bsdf &b, const V3 &v) {
    return mk(b.ss.x * v.x + b.ts.x * v.y + b.ns.x * v.z, b.ss.y * v.x + b.ts.y * v.y + b.ns.y * v.z,
              b.ss.z * v.x + b.ts.z * v.y + b.ns.z * v.z);
}
B200_HD int bsdf_num_components(const Bsdf &b, int flags) {
    int num = 0;
    for (int i = 0; i < b.n; ++i)
        if (lobe_matches(b.lobes[i], flags)) ++num;
    return num;
}
// reflection.cpp:670-683
template <int KINDS = KM_ALL>
B200_HD_L1 Spec bsdf_f(const Bsdf &b, const V3 &woW, const V3 &wiW, int flags) {
    V3 wi = world_to_local(b, wiW), wo = world_to_local(b, woW);
    if (wo.z == 0) return rgb1(0.f);
    bool refl = dot(wiW, b.ng) * dot(woW, b.ng) > 0;
    Spec f = rgb1(0.f);
    for (int i = 0; i < b.n; ++i)
        if (lobe_matches(b.lobes[i], flags) && ((refl && (b.lobes[i].type & BSDF_REFLECTION)) ||
                                                (!refl && (b.lobes[i].type & BSDF_TRANSMISSION))))
            f = f + lobe_f<KINDS>(b.lobes[i], wo, wi);
    return f;
}
// reflection.cpp:770-785
template <int KINDS = KM_ALL>
B200_HD_L1 float bsdf_pdf(const Bsdf &b, const V3 &woW, const V3 &wiW, int flags) {
    if (b.n == 0) return 0.f;
    V3 wo = world_to_local(b, woW), wi = world_to_local(b, wiW);
    if (wo.z == 0) return 0.f;
    float pdf = 0.f;
    int matching = 0;
    for (int i = 0; i < b.n; ++i)
        if (lobe_matches(b.lobes[i], flags)) {
            ++matching;
            pdf += lobe_pdf<KINDS>(b.lobes[i], wo, wi);
        }
    return matching > 0 ? pdf / matching : 0.f;
}
// reflection.cpp:703-768
template <int KINDS = KM_ALL>
B200_HD_L1 Spec bsdf_sample_f(const Bsdf &b, const V3 &woW, V3 *wiW, const float u[2], float *pdf, int type,
                          int *sampledType) {
    int matching = bsdf_num_components(b, type);
    if (matching == 0) {
        *pdf = 0;
        *sampledType = 0;
        return rgb1(0.f);
    }
    int comp_ = pt_mini((int)floorf(u[0] * matching), matching - 1);
    int which = 0, count = comp_;
    for (int i = 0; i < b.n; ++i)
        if (lobe_matches(b.lobes[i], type) && count-- == 0) {
            which = i;
            break;
        }
    const Lobe &lobe = b.lobes[which];
    float ur[2] = {pt_min(u[0] * matching - comp_, PT_ONE_MINUS_EPS), u[1]};
    V3 wi = mk(0.f, 0.f, 0.f), wo = world_to_local(b, woW);
    if (wo.z == 0) return rgb1(0.f);
    *pdf = 0;
    *sampledType = lobe.type;
    Spec f = lobe_sample_f<KINDS>(lobe, wo, &wi, ur, pdf, sampledType);
    if (*pdf == 0) {
        *sampledType = 0;
        return rgb1(0.f);
    }
    *wiW = local_to_world(b, wi);
    if (!(lobe.type & BSDF_SPECULAR) && matching > 1)
        for (int i = 0; i < b.n; ++i)
            if (i != which && lobe_matches(b.lobes[i], type)) *pdf += lobe_pdf<KINDS>(b.lobes[i], wo, wi);
    if (matching > 1) *pdf /= matching;
    if (!(lobe.type & BSDF_SPECULAR)) {
        bool refl = dot(*wiW, b.ng) * dot(woW, b.ng) > 0;
        f = rgb1(0.f);
        for (int i = 0; i < b.n; ++i)
            if (lobe_matches(b.lobes[i], type) && ((refl && (b.lobes[i].type & BSDF_REFLECTION)) ||
                                                   (!refl && (b.lobes[i].type & BSDF_TRANSMISSION))))
                f = f + lobe_f<KINDS>(b.lobes[i], wo, wi);
    }
    return f;
}

#if B200PT_NSPEC != 3
// ----------------------------------------------------------------------------------------------------------------
// Lazy spectra (SampledSpectrum build).  A 60-bin Spec by value is 240 bytes: the shading kernel that held beta, L,
// f, Li, A and B that way ran out of a 4.5-6.4 KB local-memory frame per thread.  Every spectrum
// of the path is a per-bin function of table rows and a few scalars, so the kernel keeps the *recipe* (LTerm: which
// rows, which scalars, which BxDF formula) in registers and evaluates it bin by bin, four bins at a time, straight
// from / to the per-slot arrays (slot-major, 60 floats per slot).  The per-bin arithmetic is the eager code's, operation for operation
// (lobe_f / lobe_sample_f / bsdf_f / bsdf_sample_f above, which follow core/reflection.cpp), so results are bit-identical.
enum { LT_ZERO = 0, LT_ROW_S, LT_ROW_S2, LT_MF_DIEL, LT_MF_COND, LT_MFT, LT_SPEC_R, LT_FS_R, LT_FS_T, LT_CONST };
struct LTerm {
    int op;
    const float *r;        // the lobe's R / T row; nullptr = the constant spectrum 1
    const float *eta, *k;  // LT_MF_COND: the conductor's rows
    float s0, s1, s2, s3, s4, s5;
};
B200_HD LTerm lterm_zero() {
    LTerm t;
    t.op = LT_ZERO;
    t.r = t.eta = t.k = nullptr;
    t.s0 = t.s1 = t.s2 = t.s3 = t.s4 = t.s5 = 0.f;
    return t;
}
// FrConductor (reflection.cpp:71-94) of one bin with etaI = 1; c = the clamped cosine, c2 = c*c, s2 = 1 - c2 (fr_conductor)
B200_HD float fr_conductor_bin(float c, float c2, float s2, float etat, float kk) {
    const float eta = etat / 1.f;
    const float etak = kk / 1.f;
    const float eta2 = eta * eta;
    const float etak2 = etak * etak;
    const float t0 = eta2 - etak2 - s2;
    const float a2plusb2 = sqrtf(t0 * t0 + (eta2 * 4.f) * etak2);
    const float t1 = a2plusb2 + c2;
    const float a = sqrtf((a2plusb2 + t0) * 0.5f);
    const float t2 = a * (2.f * c);
    const float Rs = (t1 - t2) / (t1 + t2);
    const float t3 = a2plusb2 * c2 + s2 * s2;
    const float t4 = t2 * s2;
    const float Rp = Rs * (t3 - t4) / (t3 + t4);
    return (Rp + Rs) * 0.5f;
}
// bins [b0, b0 + 4) of a term
template <int KINDS = KM_ALL>
B200_HD void lterm_eval4(const LTerm &t, int b0, float v[4]) {
    float x[4];
    PT_UNROLL
    for (int j = 0; j < 4; ++j) x[j] = t.r ? t.r[b0 + j] : 1.f;
    // (cases of BxDFs this family cannot have are compiled out)
    const int op = ((t.op == LT_ROW_S && !(KINDS & KM(BX_LAMBERT))) || (t.op == LT_ROW_S2 && !(KINDS & KM(BX_OREN_NAYAR))) ||
                    (t.op == LT_MF_DIEL && !(KINDS & KM_DIEL)) || (t.op == LT_MF_COND && !(KINDS & KM_COND)) ||
                    (t.op == LT_MFT && !(KINDS & KM(BX_MICROFACET_TRANS))) ||
                    (t.op == LT_SPEC_R && !(KINDS & KM(BX_SPECULAR_REFLECTION))) ||
                    ((t.op == LT_FS_R || t.op == LT_FS_T) && !(KINDS & KM(BX_FRESNEL_SPECULAR))) ||
                    (t.op == LT_CONST && !(KINDS & KM_CONST)))
                       ? LT_ZERO
                       : t.op;
    switch (op) {
    case LT_ROW_S:  // LambertianReflection::f
        if (!(KINDS & KM(BX_LAMBERT))) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = x[j] * t.s0;
        break;
    case LT_ROW_S2:  // OrenNayar::f
        if (!(KINDS & KM(BX_OREN_NAYAR))) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = (x[j] * t.s0) * t.s1;
        break;
    case LT_MF_DIEL:  // MicrofacetReflection::f with FresnelDielectric: R * D * G * F / (4 cosI cosO)
        if (!(KINDS & KM_DIEL)) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = (((x[j] * t.s0) * t.s1) * t.s2) / t.s3;
        break;
    case LT_MF_COND:  // ... with FresnelConductor
        if (!(KINDS & KM_COND)) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j)
            v[j] = (((x[j] * t.s0) * t.s1) * fr_conductor_bin(t.s2, t.s4, t.s5, t.eta[b0 + j], t.k[b0 + j])) / t.s3;
        break;
    case LT_MFT:  // MicrofacetTransmission::f: (1 - F) * T * scalar
        if (!(KINDS & KM(BX_MICROFACET_TRANS))) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = ((1.f - t.s0) * x[j]) * t.s1;
        break;
    case LT_SPEC_R:  // SpecularReflection::Sample_f with FresnelNoOp: 1 * R / |cos|
        if (!(KINDS & KM(BX_SPECULAR_REFLECTION))) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = (1.f * x[j]) / t.s0;
        break;
    case LT_FS_R:  // FresnelSpecular::Sample_f, reflection: F * R / |cos|
        if (!(KINDS & KM(BX_FRESNEL_SPECULAR))) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = (x[j] * t.s0) / t.s1;
        break;
    case LT_FS_T:  // ... transmission: T * (1 - F) * (etaI^2 / etaT^2) / |cos|
        if (!(KINDS & KM(BX_FRESNEL_SPECULAR))) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = ((x[j] * t.s0) * t.s1) / t.s2;
        break;
    case LT_CONST:  // Spectrum(p): the phase function's value at a medium vertex
        if (!(KINDS & KM_CONST)) break;
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = t.s0;
        break;
    default:
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = 0.f;
        break;
    }
}

// lobe_f as a recipe
template <int KINDS = KM_ALL>
B200_HD LTerm lobe_term(const Lobe &l, const V3 &wo, const V3 &wi) {
    LTerm t = lterm_zero();
    if ((KINDS & KM(BX_LAMBERT)) && l.kind == BX_LAMBERT) {
        t.op = LT_ROW_S;
        t.r = l.R.p;
        t.s0 = PT_INV_PI;
        return t;
    }
    if ((KINDS & KM(BX_MICROFACET)) && l.kind == BX_MICROFACET) {
        float cosThetaO = abs_cos_theta(wo), cosThetaI = abs_cos_theta(wi);
        V3 wh = wi + wo;
        if (cosThetaI == 0 || cosThetaO == 0) return t;
        if (wh.x == 0 && wh.y == 0 && wh.z == 0) return t;
        wh = normalize(wh);
        t.r = l.R.p;
        t.s0 = tr_D(l.dist, wh);
        t.s1 = tr_G(l.dist, wo, wi);
        t.s3 = 4 * cosThetaI * cosThetaO;
        const float cosF = dot(wi, wh);
        if (!(KINDS & KM_COND) || ((KINDS & KM_DIEL) && !l.conductor)) {
            t.op = LT_MF_DIEL;
            t.s2 = fr_dielectric(cosF, l.frEtaI, l.frEtaT);
        } else {
            t.op = LT_MF_COND;
            t.eta = l.cEta.p;
            t.k = l.cK.p;
            const float c = pt_clamp(pt_abs(cosF), -1.f, 1.f);
            t.s2 = c;
            t.s4 = c * c;
            t.s5 = (float)(1. - (double)t.s4);
        }
        return t;
    }
    if ((KINDS & KM(BX_OREN_NAYAR)) && l.kind == BX_OREN_NAYAR) {
        float sinThetaI = sin_theta(wi);
        float sinThetaO = sin_theta(wo);
        float maxCos = 0;
        if ((double)sinThetaI > 1e-4 && (double)sinThetaO > 1e-4) {
            float sinPhiI = sin_phi(wi), cosPhiI = cos_phi(wi);
            float sinPhiO = sin_phi(wo), cosPhiO = cos_phi(wo);
            float dCos = cosPhiI * cosPhiO + sinPhiI * sinPhiO;
            maxCos = pt_max(0.f, dCos);
        }
        float sinAlpha, tanBeta;
        if (abs_cos_theta(wi) > abs_cos_theta(wo)) {
            sinAlpha = sinThetaO;
            tanBeta = sinThetaI / abs_cos_theta(wi);
        } else {
            sinAlpha = sinThetaI;
            tanBeta = sinThetaO / abs_cos_theta(wo);
        }
        t.op = LT_ROW_S2;
        t.r = l.R.p;
        t.s0 = PT_INV_PI;
        t.s1 = l.onA + l.onB * maxCos * sinAlpha * tanBeta;
        return t;
    }
    if ((KINDS & KM(BX_MICROFACET_TRANS)) && l.kind == BX_MICROFACET_TRANS) {
        if (same_hemisphere(wo, wi)) return t;
        float cosThetaO = cos_theta(wo);
        float cosThetaI = cos_theta(wi);
        if (cosThetaI == 0 || cosThetaO == 0) return t;
        float eta = cos_theta(wo) > 0 ? (l.etaB / l.etaA) : (l.etaA / l.etaB);
        V3 wh = normalize(wo + wi * eta);
        if (wh.z < 0) wh = -wh;
        float sqrtDenom = dot(wo, wh) + eta * dot(wi, wh);
        float factor = 1 / eta;
        t.op = LT_MFT;
        t.r = l.T.p;
        t.s0 = fr_dielectric(dot(wo, wh), l.etaA, l.etaB);
        t.s1 = pt_abs(tr_D(l.dist, wh) * tr_G(l.dist, wo, wi) * eta * eta * absdot(wi, wh) * absdot(wo, wh) * factor * factor /
                      (cosThetaI * cosThetaO * sqrtDenom * sqrtDenom));
        return t;
    }
    return t;  // FresnelSpecular::f, SpecularReflection::f
}
// lobe_sample_f as a recipe
template <int KINDS = KM_ALL>
B200_HD LTerm lobe_sample_term(const Lobe &l, const V3 &wo, V3 *wi, const float u[2], float *pdf, int *sampledType) {
    LTerm t = lterm_zero();
    if ((KINDS & KM(BX_MICROFACET_TRANS)) && l.kind == BX_MICROFACET_TRANS) {
        if (wo.z == 0) return t;
        V3 wh = tr_sample_wh(l.dist, wo, u);
        float eta = cos_theta(wo) > 0 ? (l.etaA / l.etaB) : (l.etaB / l.etaA);
        if (!refract(wo, wh, eta, wi)) return t;
        *pdf = lobe_pdf<KINDS>(l, wo, *wi);
        return lobe_term<KINDS>(l, wo, *wi);
    }
    if ((KINDS & (KM(BX_LAMBERT) | KM(BX_OREN_NAYAR))) && (l.kind == BX_LAMBERT || l.kind == BX_OREN_NAYAR)) {
        *wi = cosine_sample_hemisphere(u);
        if (wo.z < 0) wi->z *= -1;
        *pdf = lobe_pdf<KINDS>(l, wo, *wi);
        return lobe_term<KINDS>(l, wo, *wi);
    }
    if ((KINDS & KM(BX_MICROFACET)) && l.kind == BX_MICROFACET) {
        if (wo.z == 0) return t;
        V3 wh = tr_sample_wh(l.dist, wo, u);
        *wi = reflect(wo, wh);
        if (!same_hemisphere(wo, *wi)) return t;
        *pdf = tr_pdf(l.dist, wo, wh) / (4 * dot(wo, wh));
        return lobe_term<KINDS>(l, wo, *wi);
    }
    if ((KINDS & KM(BX_SPECULAR_REFLECTION)) && l.kind == BX_SPECULAR_REFLECTION) {
        *wi = mk(-wo.x, -wo.y, wo.z);
        *pdf = 1.f;
        t.op = LT_SPEC_R;
        t.r = l.R.p;
        t.s0 = abs_cos_theta(*wi);
        return t;
    }
    if (!(KINDS & KM(BX_FRESNEL_SPECULAR))) return t;
    float F = fr_dielectric(cos_theta(wo), l.etaA, l.etaB);
    if (u[0] < F) {
        *wi = mk(-wo.x, -wo.y, wo.z);
        *sampledType = BSDF_SPECULAR | BSDF_REFLECTION;
        *pdf = F;
        t.op = LT_FS_R;
        t.r = l.R.p;
        t.s0 = F;
        t.s1 = abs_cos_theta(*wi);
        return t;
    }
    bool entering = cos_theta(wo) > 0;
    float etaI = entering ? l.etaA : l.etaB;
    float etaT = entering ? l.etaB : l.etaA;
    V3 nn = mk(0.f, 0.f, 1.f);
    if (dot(nn, wo) < 0.f) nn = -nn;
    if (!refract(wo, nn, etaI / etaT, wi)) return t;
    *sampledType = BSDF_SPECULAR | BSDF_TRANSMISSION;
    *pdf = 1 - F;
    t.op = LT_FS_T;
    t.r = l.T.p;
    t.s0 = 1 - F;
    t.s1 = (etaI * etaI) / (etaT * etaT);
    t.s2 = abs_cos_theta(*wi);
    return t;
}
// A BSDF value: the sum (in lobe order, starting from 0 like `Spectrum f(0.f); f += ...` when from_zero) of up to two terms
struct FSpec {
    int n;
    int from_zero;
    LTerm t[2];
};
B200_HD FSpec fspec_zero() {
    FSpec f;
    f.n = 0;
    f.from_zero = 1;
    f.t[0] = f.t[1] = lterm_zero();
    return f;
}
B200_HD FSpec fspec_const(float p) {
    FSpec f = fspec_zero();
    f.n = 1;
    f.from_zero = 0;
    f.t[0].op = LT_CONST;
    f.t[0].s0 = p;
    return f;
}
template <int KINDS = KM_ALL>
B200_HD_S60 void fspec_eval4(const FSpec &f, int b0, float v[4]) {
    if (f.n == 0) {
        v[0] = v[1] = v[2] = v[3] = 0.f;
        return;
    }
    lterm_eval4<KINDS>(f.t[0], b0, v);
    if (f.from_zero) {
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = 0.f + v[j];
    }
    if (f.n > 1) {
        float w[4];
        lterm_eval4<KINDS>(f.t[1], b0, w);
        PT_UNROLL
        for (int j = 0; j < 4; ++j) v[j] = v[j] + w[j];
    }
}
// is_black(f * s) without materialising it
template <int KINDS = KM_ALL>
B200_HD bool fspec_is_black(const FSpec &f, float s) {
    if (f.n == 0) return true;
    for (int b0 = 0; b0 < B200PT_NSPEC; b0 += 4) {
        float v[4];
        fspec_eval4<KINDS>(f, b0, v);
        if (v[0] * s != 0.f || v[1] * s != 0.f || v[2] * s != 0.f || v[3] * s != 0.f) return false;
    }
    return true;
}
B200_HD bool row_is_black(const float *p) {
    for (int i = 0; i < B200PT_NSPEC; ++i)
        if (p[i] != 0.f) return false;
    return true;
}
// bsdf_f (reflection.cpp:670-683) as a recipe
template <int KINDS = KM_ALL>
B200_HD_L1 FSpec bsdf_f_lazy(const Bsdf &b, const V3 &woW, const V3 &wiW, int flags) {
    FSpec f = fspec_zero();
    V3 wi = world_to_local(b, wiW), wo = world_to_local(b, woW);
    if (wo.z == 0) return f;
    bool refl = dot(wiW, b.ng) * dot(woW, b.ng) > 0;
    for (int i = 0; i < b.n; ++i)
        if (lobe_matches(b.lobes[i], flags) && ((refl && (b.lobes[i].type & BSDF_REFLECTION)) ||
                                                (!refl && (b.lobes[i].type & BSDF_TRANSMISSION))))
            f.t[f.n++] = lobe_term<KINDS>(b.lobes[i], wo, wi);
    return f;
}
// bsdf_sample_f (reflection.cpp:703-768) as a recipe
template <int KINDS = KM_ALL>
B200_HD_L1 FSpec bsdf_sample_f_lazy(const Bsdf &b, const V3 &woW, V3 *wiW, const float u[2], float *pdf, int type, int *sampledType) {
    FSpec f = fspec_zero();
    int matching = bsdf_num_components(b, type);
    if (matching == 0) {
        *pdf = 0;
        *sampledType = 0;
        return f;
    }
    int comp_ = pt_mini((int)floorf(u[0] * matching), matching - 1);
    int which = 0, count = comp_;
    for (int i = 0; i < b.n; ++i)
        if (lobe_matches(b.lobes[i], type) && count-- == 0) {
            which = i;
            break;
        }
    const Lobe &lobe = b.lobes[which];
    float ur[2] = {pt_min(u[0] * matching - comp_, PT_ONE_MINUS_EPS), u[1]};
    V3 wi = mk(0.f, 0.f, 0.f), wo = world_to_local(b, woW);
    if (wo.z == 0) return f;
    *pdf = 0;
    *sampledType = lobe.type;
    const LTerm ts = lobe_sample_term<KINDS>(lobe, wo, &wi, ur, pdf, sampledType);
    if (*pdf == 0) {
        *sampledType = 0;
        return f;
    }
    *wiW = local_to_world(b, wi);
    if (!(lobe.type & BSDF_SPECULAR) && matching > 1)
        for (int i = 0; i < b.n; ++i)
            if (i != which && lobe_matches(b.lobes[i], type)) *pdf += lobe_pdf<KINDS>(b.lobes[i], wo, wi);
    if (matching > 1) *pdf /= matching;
    if (!(lobe.type & BSDF_SPECULAR)) {
        bool refl = dot(*wiW, b.ng) * dot(woW, b.ng) > 0;
        for (int i = 0; i < b.n; ++i)
            if (lobe_matches(b.lobes[i], type) && ((refl && (b.lobes[i].type & BSDF_REFLECTION)) ||
                                                   (!refl && (b.lobes[i].type & BSDF_TRANSMISSION))))
                f.t[f.n++] = lobe_term<KINDS>(b.lobes[i], wo, wi);
    } else {
        f.n = 1;
        f.from_zero = 0;
        f.t[0] = ts;
    }
    return f;
}
#endif  // B200PT_NSPEC != 3

B200_HD void add_lambert(Bsdf *b, const float *kd) {
    Lobe &l = b->lobes[b->n++];
    l.kind = BX_LAMBERT;
    l.type = BSDF_REFLECTION | BSDF_DIFFUSE;
    l.R = sref(kd);
}
// Material::ComputeScatteringFunctions with constant textures
// (allowMultipleLobes = true, TransportMode::Radiance; path.cpp:107).
// MATERIAL is a b200pt_material_type known at compile time in the per-family
// shading kernels, or -1 for a run-time switch.
// The spectra of a material: the descriptor's RGB triples, or (SampledSpectrum build) the material's rows of
// b200pt_scene_desc::material_spectra, B200PT_MATERIAL_SPECTRA rows of 60 bins in the order kd, ks, kt, eta, k.
struct MatSpec {
    const float *kd, *ks, *kt, *eta, *k;
};
B200_HD MatSpec mat_spec(const b200pt_material &m, const float *rows) {
    MatSpec s;
#if B200PT_NSPEC == 3
    (void)rows;
    s.kd = m.kd;
    s.ks = m.ks;
    s.kt = m.kt;
    s.eta = m.eta;
    s.k = m.k;
#else
    s.kd = rows;
    s.ks = rows + B200PT_NSPEC;
    s.kt = rows + 2 * B200PT_NSPEC;
    s.eta = rows + 3 * B200PT_NSPEC;
    s.k = rows + 4 * B200PT_NSPEC;
#endif
    return s;
}
// is_black of a material row (the 60-bin build tests the row in place instead of copying it)
#if B200PT_NSPEC == 3
#define PT_ROW_BLACK(p) is_black(rgbp(p))
#else
#define PT_ROW_BLACK(p) row_is_black(p)
#endif
template <int MATERIAL>
B200_HD void make_bsdf(const b200pt_material &m, const float *spectra_rows, const Isect &is, Bsdf *b) {
    const MatSpec ms = mat_spec(m, spectra_rows);
    b->eta = 1.f;
    b->ns = is.ns;  // reflection.h:157
    b->ng = is.n;
    b->ss = normalize(is.sdpdu);  // reflection.h:159
    b->ts = cross(b->ns, b->ss);  // reflection.h:160
    b->n = 0;
    const int type = MATERIAL >= 0 ? MATERIAL : m.type;
    if (type == B200PT_MAT_MATTE) {  // matte.cpp:45-62
        if (!PT_ROW_BLACK(ms.kd)) {
            add_lambert(b, ms.kd);
            if (m.variant == 1) {  // sigma != 0: OrenNayar(r, sig)
                Lobe &l = b->lobes[b->n - 1];
                l.kind = BX_OREN_NAYAR;
                l.onA = m.alpha_x;
                l.onB = m.alpha_y;
            }
        }
    } else if (type == B200PT_MAT_PLASTIC) {  // plastic.cpp:45-70
        if (!PT_ROW_BLACK(ms.kd)) add_lambert(b, ms.kd);
        if (!PT_ROW_BLACK(ms.ks)) {
            Lobe &l = b->lobes[b->n++];
            l.kind = BX_MICROFACET;
            l.type = BSDF_REFLECTION | BSDF_GLOSSY;
            l.R = sref(ms.ks);
            l.dist.ax = m.alpha_x;
            l.dist.ay = m.alpha_x;
            l.conductor = 0;
            l.frEtaI = 1.5f;
            l.frEtaT = 1.f;
        }
    } else if (type == B200PT_MAT_METAL) {  // metal.cpp:59-80
        Lobe &l = b->lobes[b->n++];
        l.kind = BX_MICROFACET;
        l.type = BSDF_REFLECTION | BSDF_GLOSSY;
        l.R = sref_one();
        l.dist.ax = m.alpha_x;
        l.dist.ay = m.alpha_y;
        l.conductor = 1;
        l.cEta = sref(ms.eta);
        l.cK = sref(ms.k);
    } else if (type == B200PT_MAT_GLASS && m.variant == 2) {  // MirrorMaterial, mirror.cpp:45-56 (BSDF eta stays 1)
        if (!PT_ROW_BLACK(ms.ks)) {
            Lobe &l = b->lobes[b->n++];
            l.kind = BX_SPECULAR_REFLECTION;
            l.type = BSDF_REFLECTION | BSDF_SPECULAR;
            l.R = sref(ms.ks);
        }
    } else if (type == B200PT_MAT_GLASS) {  // glass.cpp:45-64
        b->eta = m.index;
        const bool blackR = PT_ROW_BLACK(ms.ks), blackT = PT_ROW_BLACK(ms.kt);
        if (blackR && blackT) {
        } else if (m.variant == 1) {  // rough glass, glass.cpp:65-90
            if (!blackR) {
                Lobe &l = b->lobes[b->n++];
                l.kind = BX_MICROFACET;
                l.type = BSDF_REFLECTION | BSDF_GLOSSY;
                l.R = sref(ms.ks);
                l.dist.ax = m.alpha_x;
                l.dist.ay = m.alpha_y;
                l.conductor = 0;
                l.frEtaI = 1.f;
                l.frEtaT = m.index;
            }
            if (!blackT) {
                Lobe &l = b->lobes[b->n++];
                l.kind = BX_MICROFACET_TRANS;
                l.type = BSDF_TRANSMISSION | BSDF_GLOSSY;
                l.T = sref(ms.kt);
                l.dist.ax = m.alpha_x;
                l.dist.ay = m.alpha_y;
                l.etaA = 1.f;
                l.etaB = m.index;
            }
        } else {
            Lobe &l = b->lobes[b->n++];
            l.kind = BX_FRESNEL_SPECULAR;
            l.type = BSDF_REFLECTION | BSDF_TRANSMISSION | BSDF_SPECULAR;
            l.R = sref(ms.ks);
            l.T = sref(ms.kt);
            l.etaA = 1.f;
            l.etaB = m.index;
        }
    }
}

// --------------------------------------------------------------------- lights
struct LightSample {
    V3 p, n, pError;
};
// shapes/triangle.cpp:583-608 + sampling.cpp:154-157
B200_HD LightSample triangle_sample(const V3 &p0, const V3 &p1, const V3 &p2, bool flip, const TriShading &sh,
                                    const float u[2], float *pdf) {
    float su0 = sqrtf(u[0]);
    float b0 = 1 - su0, b1 = u[1] * su0;
    LightSample it;
    it.p = b0 * p0 + b1 * p1 + (1 - b0 - b1) * p2;
    it.n = normalize(cross(p1 - p0, p2 - p0));
    if (sh.has_n) {
        const V3 ns = b0 * sh.n0 + b1 * sh.n1 + (1 - b0 - b1) * sh.n2;
        it.n = (dot(it.n, ns) < 0.f) ? -it.n : it.n;  // Faceforward, triangle.cpp:596-600
    } else if (flip)
        it.n = it.n * -1.f;
    V3 s = vabs(b0 * p0) + vabs(b1 * p1) + vabs((1 - b0 - b1) * p2);
    it.pError = pt_gamma(6) * mk(s.x, s.y, s.z);
    *pdf = 1 / triangle_area(p0, p1, p2);
    return it;
}
// sampling.h:171-174
B200_HD float power_heuristic(float fPdf, float gPdf) {
    float f = fPdf, g = gPdf;
    return (f * f) / (f * f + g * g);
}
// pbrt.h:353-368 FindInterval over cdf[0..size-1] with the predicate cdf[i] <= u
B200_HD int find_interval(const float *cdf, int size, float u) {
    int first = 0, l = size;
    while (l > 0) {
        int half = l >> 1, middle = first + half;
        if (cdf[middle] <= u) {
            first = middle + 1;
            l -= half + 1;
        } else
            l = half;
    }
    return pt_mini(pt_maxi(first - 1, 0), size - 2);
}
// sampling.h:90-100 over cdf[0..n]
B200_HD int sample_discrete(const float *cdf, const float *func, float funcInt, int n, float u, float *pdf) {
    int offset = find_interval(cdf, n + 1, u);
    *pdf = (funcInt > 0) ? func[offset] / (funcInt * n) : 0.f;
    return offset;
}

// ------------------------------------------------ spatial light distribution
// core/lowdiscrepancy.cpp:389-403, 427-444 (RadicalInverse for bases 2, 3, 5, 7, 11)
B200_HD uint32_t reverse_bits32(uint32_t n) {
    n = (n << 16) | (n >> 16);
    n = ((n & 0x00ff00ffu) << 8) | ((n & 0xff00ff00u) >> 8);
    n = ((n & 0x0f0f0f0fu) << 4) | ((n & 0xf0f0f0f0u) >> 4);
    n = ((n & 0x33333333u) << 2) | ((n & 0xccccccccu) >> 2);
    n = ((n & 0x55555555u) << 1) | ((n & 0xaaaaaaaau) >> 1);
    return n;
}
B200_HD float radical_inverse(int baseIndex, uint64_t a) {
    if (baseIndex == 0) {
        const uint64_t n0 = reverse_bits32((uint32_t)a), n1 = reverse_bits32((uint32_t)(a >> 32));
        return (float)((double)((n0 << 32) | n1) * 0x1p-64);
    }
    const int base = baseIndex == 1 ? 3 : (baseIndex == 2 ? 5 : (baseIndex == 3 ? 7 : 11));
    const float invBase = 1.0f / (float)base;
    uint64_t reversedDigits = 0;
    float invBaseN = 1;
    while (a) {
        const uint64_t next = a / (uint64_t)base;
        const uint64_t digit = a - next * (uint64_t)base;
        reversedDigits = reversedDigits * (uint64_t)base + digit;
        invBaseN *= invBase;
        a = next;
    }
    return pt_min((float)reversedDigits * invBaseN, PT_ONE_MINUS_EPS);
}
B200_HD float lerpf(float t, float v1, float v2) { return (1 - t) * v1 + t * v2; }  // pbrt.h:413

struct SpatialGrid {        // SpatialLightDistribution, lightdistrib.cpp:96-124
    int enabled;
    int nv[3];
    float wb_min[3], wb_max[3];  // Scene::WorldBound()
};
// SpatialLightDistribution::Lookup, lightdistrib.cpp:139-148: voxel of a point
B200_HD int spatial_voxel(const SpatialGrid &g, const V3 &p) {
    int pi[3];
    const float pc[3] = {p.x, p.y, p.z};
    for (int a = 0; a < 3; ++a) {
        float o = pc[a] - g.wb_min[a];
        if (g.wb_max[a] > g.wb_min[a]) o /= g.wb_max[a] - g.wb_min[a];
        const int v = (int)(o * (float)g.nv[a]);
        pi[a] = v < 0 ? 0 : (v > g.nv[a] - 1 ? g.nv[a] - 1 : v);
    }
    return (pi[2] * g.nv[1] + pi[1]) * g.nv[0] + pi[0];
}
// One (voxel, light) term of SpatialLightDistribution::ComputeDistribution (lightdistrib.cpp:230-275):
// sum over 128 Halton points of Li.y()/pdf for a DiffuseAreaLight on the triangle (p0,p1,p2).
// spatial_light_contrib: see pt_sphere.cuh (it samples triangle and sphere lights)

// --------------------------------------------------------------------- media
#define PT_MAX_FLOAT 3.402823466e+38f
#define PT_INV_4PI ((float)0.07957747154594766788)
// Exp(-sigma_t * x) per bin (spectrum.h:217-227 with the host's expf, pt_explog.cuh)
B200_HD Spec spec_exp_neg(const Spec &sigma_t, float x) {
    Spec r;
    PT_UNROLL SPEC_FOR r.c[i_] = pt_expf((-sigma_t.c[i_]) * x);
    return r;
}
// HomogeneousMedium::Tr (homogeneous.cpp:44-47) of a ray (d, tMax)
B200_HD Spec medium_tr(const Spec &sigma_t, const V3 &d, float tMax) { return spec_exp_neg(sigma_t, pt_min(tMax * len(d), PT_MAX_FLOAT)); }
// medium.h:69-72
B200_HD float phase_hg(float cosTheta, float g) {
    float denom = 1 + g * g + 2 * g * cosTheta;
    return PT_INV_4PI * (1 - g * g) / (denom * sqrtf(denom));
}
// HenyeyGreenstein::Sample_p, medium.cpp:194-213
B200_HD float hg_sample_p(float g, const V3 &wo, V3 *wi, const float u[2]) {
    float cosTheta;
    if (pt_abs(g) < 1e-3)
        cosTheta = 1 - 2 * u[0];
    else {
        float sqrTerm = (1 - g * g) / (1 - g + 2 * g * u[0]);
        cosTheta = (1 + g * g - sqrTerm * sqrTerm) / (2 * g);
    }
    float sinTheta = sqrtf(pt_max(0.f, 1 - cosTheta * cosTheta));
    float phi = 2 * PT_PI * u[1];
    V3 v1, v2;
    coordinate_system(wo, &v1, &v2);
    // SphericalDirection(sinTheta, cosTheta, phi, v1, v2, -wo), geometry.h:1467-1472
    *wi = v1 * (sinTheta * pt_cosf(phi)) + v2 * (sinTheta * pt_sinf(phi)) + (-wo) * cosTheta;
    return phase_hg(-cosTheta, g);
}

// ----------------------------------------------------------------------- film
// Spectrum::ToXYZ: RGBSpectrum (spectrum.h:455 -> :62-66) or SampledSpectrum (spectrum.h:380-392)
B200_HD void rgb_to_xyz(const Spec &c, float xyz[3]) {
#if B200PT_NSPEC == 3
    xyz[0] = 0.412453f * c.c[0] + 0.357580f * c.c[1] + 0.180423f * c.c[2];
    xyz[1] = 0.212671f * c.c[0] + 0.715160f * c.c[1] + 0.072169f * c.c[2];
    xyz[2] = 0.019334f * c.c[0] + 0.119193f * c.c[1] + 0.950227f * c.c[2];
#else
    xyz[0] = xyz[1] = xyz[2] = 0.f;
    SPEC_FOR {
        xyz[0] += PT_CIE(0, i_) * c.c[i_];
        xyz[1] += PT_CIE(1, i_) * c.c[i_];
        xyz[2] += PT_CIE(2, i_) * c.c[i_];
    }
    const float scale = PT_SPECTRAL_SCALE;
    xyz[0] *= scale;
    xyz[1] *= scale;
    xyz[2] *= scale;
#endif
}
B200_HD void xyz_to_rgb(const float xyz[3], float rgbv[3]) {  // spectrum.h:56-60
    rgbv[0] = 3.240479f * xyz[0] - 1.537150f * xyz[1] - 0.498535f * xyz[2];
    rgbv[1] = -0.969256f * xyz[0] + 1.875991f * xyz[1] + 0.041556f * xyz[2];
    rgbv[2] = 0.055648f * xyz[0] - 0.204043f * xyz[1] + 1.057311f * xyz[2];
}

}  // namespace B200PT_NS
#endif
