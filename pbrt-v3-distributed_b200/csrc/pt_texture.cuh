// pt_texture.cuh -- ImageTexture's MIPMap lookups, RoughnessToAlpha and InfiniteAreaLight's Le / Sample_Li / Pdf_Li
// over the tables the host copied from the reference's own MIPMap and Distribution2D (kernels.cuh: DevMipmap,
// DevInfinite).  __host__ __device__, so that the test harness (tests/devmath) can run the same code host-compiled;
// kernels.cu calls them from the shading and escaped-ray kernels.  RGBSpectrum build only.
#ifndef B200PT_TEXTURE_CUH
#define B200PT_TEXTURE_CUH

#include "kernels.cuh"

#if B200PT_NSPEC == 3
namespace B200PT_NS {

// ---- InfiniteAreaLight (lights/infinite.cpp:92-132) over the host's level-0 texels and Distribution2D tables
#define PT_INV_PI ((float)0.31830988618379067154)
#define PT_INV_2PI ((float)0.15915494309189533577)
// Mod (pbrt.h)
__host__ __device__ __forceinline__ int pt_mod(int a, int b) {
    const int r = a - (a / b) * b;
    return r < 0 ? r + b : r;
}
// MIPMap::triangle(level, st) (mipmap.h:262-273) on a level of w x h texels: bilinear, the weights formed first;
// texel(s, t) is MIPMap::Texel with the map's wrap mode
template <class Texel>
__host__ __device__ __forceinline__ Spec mip_bilerp(int w, int h, float st0, float st1, const Texel &texel) {
    const float s = st0 * w - 0.5f, t = st1 * h - 0.5f;
    const int s0 = (int)floorf(s), t0 = (int)floorf(t);
    const float ds = s - s0, dt = t - t0;
    return (1 - ds) * (1 - dt) * texel(s0, t0) + (1 - ds) * dt * texel(s0, t0 + 1) + ds * (1 - dt) * texel(s0 + 1, t0) +
           ds * dt * texel(s0 + 1, t0 + 1);
}
// MIPMap::triangle(0, st) of the sky: Repeat wrap
__host__ __device__ __forceinline__ Spec infinite_lookup(const DevInfinite &L, float st0, float st1) {
    return mip_bilerp(L.w, L.h, st0, st1, [&](int si, int ti) {
        const float4 v = L.texels[(size_t)pt_mod(ti, L.h) * L.w + pt_mod(si, L.w)];
        return rgb(v.x, v.y, v.z);
    });
}

// ---- ImageTexture lookups: MIPMap (mipmap.h:220-353) on RGB texels; a float map runs the same arithmetic on x
// MIPMap::Texel (mipmap.h:220-242)
__host__ __device__ __forceinline__ Spec mip_texel(const DevMipmap &M, int level, int s, int t) {
    const int w = M.w[level], h = M.h[level];
    if (M.wrap == B200PT_WRAP_REPEAT) {
        s = pt_mod(s, w);
        t = pt_mod(t, h);
    } else if (M.wrap == B200PT_WRAP_CLAMP) {
        s = pt_mini(pt_maxi(s, 0), w - 1);
        t = pt_mini(pt_maxi(t, 0), h - 1);
    } else if (s < 0 || s >= w || t < 0 || t >= h) {
        return rgb1(0.f);
    }
    const float4 v = M.texels[level][(size_t)t * w + s];
    return rgb(v.x, v.y, v.z);
}
__host__ __device__ __forceinline__ Spec mip_triangle(const DevMipmap &M, int level, float st0, float st1) {
    level = pt_mini(pt_maxi(level, 0), M.levels - 1);
    return mip_bilerp(M.w[level], M.h[level], st0, st1, [&](int si, int ti) { return mip_texel(M, level, si, ti); });
}
__host__ __device__ __forceinline__ float pt_log2f(float x) { return pt_logf(x) * 1.442695040888963387004650940071f; }  // Log2, pbrt.h
__host__ __device__ __forceinline__ Spec mip_lerp(float t, const Spec &a, const Spec &b) { return (1 - t) * a + t * b; }
// MIPMap::Lookup(st, width) (mipmap.h:244-261)
__host__ __device__ __forceinline__ Spec mip_lookup_width(const DevMipmap &M, float st0, float st1, float width) {
    const float level = M.levels - 1 + pt_log2f(pt_max(width, (float)1e-8));
    if (level < 0) return mip_triangle(M, 0, st0, st1);
    if (level >= M.levels - 1) return mip_texel(M, M.levels - 1, 0, 0);
    const int iLevel = (int)floorf(level);
    const float delta = level - iLevel;
    return mip_lerp(delta, mip_triangle(M, iLevel, st0, st1), mip_triangle(M, iLevel + 1, st0, st1));
}
// MIPMap::EWA (mipmap.h:305-353)
__host__ __device__ Spec mip_ewa(const DevMipmap &M, int level, float st0, float st1, float d00, float d01, float d10, float d11) {
    if (level >= M.levels) return mip_texel(M, M.levels - 1, 0, 0);
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
    const int s0 = (int)ceilf(st0 - 2 * invDet * uSqrt);
    const int s1 = (int)floorf(st0 + 2 * invDet * uSqrt);
    const int t0 = (int)ceilf(st1 - 2 * invDet * vSqrt);
    const int t1 = (int)floorf(st1 + 2 * invDet * vSqrt);
    Spec sum = rgb1(0.f);
    float sumWts = 0;
    for (int it = t0; it <= t1; ++it) {
        const float tt = it - st1;
        for (int is = s0; is <= s1; ++is) {
            const float ss = is - st0;
            const float r2 = A * ss * ss + B * ss * tt + C * tt * tt;
            if (r2 < 1) {
                const int index = pt_mini((int)(r2 * 128), 128 - 1);
                const float weight = M.weight_lut[index];
                sum = sum + mip_texel(M, level, is, it) * weight;
                sumWts += weight;
            }
        }
    }
    return sum / sumWts;
}
// MIPMap::Lookup(st, dst0, dst1) (mipmap.h:276-303)
__host__ __device__ Spec mip_lookup(const DevMipmap &M, float st0, float st1, float d00, float d01, float d10, float d11) {
    if (M.trilinear) {
        const float width = pt_max(pt_max(pt_abs(d00), pt_abs(d01)), pt_max(pt_abs(d10), pt_abs(d11)));
        return mip_lookup_width(M, st0, st1, 2 * width);
    }
    if (d00 * d00 + d01 * d01 < d10 * d10 + d11 * d11) {
        float t = d00;
        d00 = d10;
        d10 = t;
        t = d01;
        d01 = d11;
        d11 = t;
    }
    const float majorLength = sqrtf(d00 * d00 + d01 * d01);
    float minorLength = sqrtf(d10 * d10 + d11 * d11);
    if (minorLength * M.max_aniso < majorLength && minorLength > 0) {
        const float scale = majorLength / (minorLength * M.max_aniso);
        d10 *= scale;
        d11 *= scale;
        minorLength *= scale;
    }
    if (minorLength == 0) return mip_triangle(M, 0, st0, st1);
    const float lod = pt_max((float)0, M.levels - (float)1 + pt_log2f(minorLength));
    const int ilod = (int)floorf(lod);
    return mip_lerp(lod - ilod, mip_ewa(M, ilod, st0, st1, d00, d01, d10, d11), mip_ewa(M, ilod + 1, st0, st1, d00, d01, d10, d11));
}
// TrowbridgeReitzDistribution::RoughnessToAlpha (microfacet.h:123-128)
__host__ __device__ __forceinline__ float roughness_to_alpha(float roughness) {
    roughness = pt_max(roughness, (float)1e-3);
    const float x = pt_logf(roughness);
    return 1.62142f + 0.819955f * x + 0.1734f * x * x + 0.0171201f * x * x * x + 0.000640711f * x * x * x * x;
}
// Spectrum::Clamp() (spectrum.h:256-262, low 0, high Infinity)
__host__ __device__ __forceinline__ void clamp_rgb(const Spec &v, float out[3]) {
    for (int c = 0; c < 3; ++c) out[c] = v.c[c] < 0.f ? 0.f : (v.c[c] > pt_inf() ? pt_inf() : v.c[c]);
}
// SphericalPhi (geometry.h:1478-1481)
__host__ __device__ __forceinline__ float spherical_phi(const V3 &v) {
    const float p = pt_atan2f(v.y, v.x);
    return (p < 0) ? (p + 2 * PT_PI) : p;
}
// InfiniteAreaLight::Le (infinite.cpp:92-96)
__host__ __device__ __forceinline__ Spec infinite_le(const DevInfinite &L, const V3 &d) {
    const V3 w = normalize(xform_vector(L.world_to_light, d));
    return infinite_lookup(L, spherical_phi(w) * PT_INV_2PI, pt_acosf(pt_clamp(w.z, -1.f, 1.f)) * PT_INV_PI);
}
// Distribution1D::SampleContinuous (sampling.h:71-89) over func[n], cdf[n + 1]
__host__ __device__ __forceinline__ float dist1d_sample(const float *func, const float *cdf, float funcInt, int n, float u, float *pdf, int *off) {
    const int offset = find_interval(cdf, n + 1, u);
    *off = offset;
    float du = u - cdf[offset];
    if ((cdf[offset + 1] - cdf[offset]) > 0) du /= (cdf[offset + 1] - cdf[offset]);
    *pdf = (funcInt > 0) ? func[offset] / funcInt : 0;
    return (offset + du) / n;
}
// InfiniteAreaLight::Sample_Li (infinite.cpp:98-122) with Distribution2D::SampleContinuous (sampling.h:124-131); *pdf stays 0
// when the map's pdf is 0.  *pTarget: the point the VisibilityTester aims at.
__host__ __device__ __forceinline__ Spec infinite_sample_li(const DevInfinite &L, const V3 &refP, const float u[2], V3 *wi, float *pdf,
                                                   V3 *pTarget) {
    *pdf = 0.f;
    *wi = *pTarget = mk(0.f, 0.f, 0.f);
    float pdfs[2];
    int v, iu;
    const float d1 = dist1d_sample(L.marg_func, L.marg_cdf, L.marg_func_int, L.nv, u[1], &pdfs[1], &v);
    const float d0 = dist1d_sample(L.cond_func + (size_t)v * L.nu, L.cond_cdf + (size_t)v * (L.nu + 1), L.cond_func_int[v], L.nu, u[0],
                                   &pdfs[0], &iu);
    const float mapPdf = pdfs[0] * pdfs[1];
    if (mapPdf == 0) return rgb1(0.f);
    const float theta = d1 * PT_PI, phi = d0 * 2 * PT_PI;
    const float cosTheta = pt_cosf(theta), sinTheta = pt_sinf(theta);
    const float sinPhi = pt_sinf(phi), cosPhi = pt_cosf(phi);
    *wi = xform_vector(L.light_to_world, mk(sinTheta * cosPhi, sinTheta * sinPhi, cosTheta));
    *pdf = mapPdf / (2 * PT_PI * PT_PI * sinTheta);
    if (sinTheta == 0) *pdf = 0;
    *pTarget = refP + *wi * L.two_world_radius;
    return infinite_lookup(L, d0, d1);
}
// InfiniteAreaLight::Pdf_Li (infinite.cpp:124-132; the direction is not normalised) with Distribution2D::Pdf (sampling.h:132-139)
__host__ __device__ __forceinline__ float infinite_pdf_li(const DevInfinite &L, const V3 &w) {
    const V3 wi = xform_vector(L.world_to_light, w);
    const float theta = pt_acosf(pt_clamp(wi.z, -1.f, 1.f)), phi = spherical_phi(wi);
    const float sinTheta = pt_sinf(theta);
    if (sinTheta == 0) return 0;
    const float p0 = phi * PT_INV_2PI, p1 = theta * PT_INV_PI;
    const int iu = pt_mini(pt_maxi(int(p0 * L.nu), 0), L.nu - 1);
    const int iv = pt_mini(pt_maxi(int(p1 * L.nv), 0), L.nv - 1);
    return L.cond_func[(size_t)iv * L.nu + iu] / L.marg_func_int / (2 * PT_PI * PT_PI * sinTheta);
}

}  // namespace B200PT_NS
#endif  // B200PT_NSPEC == 3
#endif
