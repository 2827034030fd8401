// pt_sphere.cuh -- the Sphere shape of the reference on the device
// (shapes/sphere.cpp:49-306), full or clipped by zmin / zmax / phimax.
//
// A sphere keeps its object space: rays are transformed with the reference's
// error-tracking Transform operators (core/transform.h:278-384), the quadratic
// is solved in EFloat interval arithmetic (core/efloat.h:47-285) because the
// choice between the two roots and the tMax test read the interval bounds, and
// the hit is transformed back with Transform::operator()(SurfaceInteraction)
// (core/transform.cpp:262-297).  std::acos is restated from the host libm the
// reference calls (glibc's fdlibm-derived float routine; pinned exhaustively
// over [-1, 1] by tests/host_preflight.cpp); std::sin / std::cos come from
// pt_sincos.cuh.  std::atan2 (restated the same way) is evaluated only for
// spheres clipped by zmin / zmax / phimax: for a full sphere phi can never exceed
// phiMax and otherwise only feeds the (u, v) of constant textures.
//
// Spheres are few (lights, a handful of objects) and are tested outside the
// triangle BVH by k_spheres after each traversal launch, with tMax already
// shortened by the triangle hit.
#ifndef B200PT_SPHERE_CUH
#define B200PT_SPHERE_CUH

#include "pt_core.cuh"
#include "pt_sincos.cuh"
#include "wbvh.h"

namespace B200PT_NS {

// hit ids >= SPHERE_HIT_BASE (and != B200PT_MISS) name sphere (id & SPHERE_HIT_MASK)
#define SPHERE_HIT_BASE 0xC0000000u
#define SPHERE_HIT_MASK 0x3fffffffu
B200_HD bool is_sphere_hit(uint32_t id) { return id >= SPHERE_HIT_BASE && id != 0xffffffffu; }

struct DevSphere {
    float o2w[16], w2o[16];  // ObjectToWorld->m, WorldToObject->m (= ObjectToWorld->mInv)
    float radius;
    float phi_max;           // Sphere::phiMax (radians); Radians(360) for a full sphere
    float theta_min, theta_max;  // Sphere::thetaMin / thetaMax; acos(-1), acos(1) for a full sphere
    float z_min, z_max;      // Sphere::zMin / zMax; -r, r for a full sphere
    float area;              // Sphere::Area(), sphere.cpp:207
    uint32_t mat_flags;      // material id | B200PT_TRI_FLIP (reverseOrientation ^ transformSwapsHandedness)
    int light_id;
    int reverse_orientation;
    float leaf_lo[3], leaf_hi[3];  // bounds of the host accelerator's leaf holding the sphere (b200pt_sphere::leaf_bounds)
};

// ---- glibc 2.3x acosf (sysdeps/ieee754/flt-32/e_acosf.c, fdlibm): float arithmetic only
B200_HD float pt_acosf(float x) {
    const float one = 1.0f, pi = 3.1415925026e+00f, pio2_hi = 1.5707962513e+00f, pio2_lo = 7.5497894159e-08f,
                pS0 = 1.6666667163e-01f, pS1 = -3.2556581497e-01f, pS2 = 2.0121252537e-01f, pS3 = -4.0055535734e-02f,
                pS4 = 7.9153501429e-04f, pS5 = 3.4793309169e-05f, qS1 = -2.4033949375e+00f, qS2 = 2.0209457874e+00f,
                qS3 = -6.8828397989e-01f, qS4 = 7.7038154006e-02f;
    float z, p, q, r, w, s, c, df;
    const int32_t hx = (int32_t)float_as_uint(x), ix = hx & 0x7fffffff;
    if (ix == 0x3f800000) {
        if (hx > 0) return 0.0f;
        return pi + 2.0f * pio2_lo;
    } else if (ix > 0x3f800000) {
        return (x - x) / (x - x);
    }
    if (ix < 0x3f000000) {
        if (ix <= 0x32800000) return pio2_hi + pio2_lo;
        z = x * x;
        p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
        q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
        r = p / q;
        return pio2_hi - (x - (pio2_lo - x * r));
    } else if (hx < 0) {
        z = (one + x) * 0.5f;
        p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
        q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
        s = sqrtf(z);
        r = p / q;
        w = r * s - pio2_lo;
        return pi - 2.0f * (s + w);
    } else {
        z = (one - x) * 0.5f;
        s = sqrtf(z);
        df = uint_as_float(float_as_uint(s) & 0xfffff000u);
        c = (z - df * df) / (s + df);
        p = z * (pS0 + z * (pS1 + z * (pS2 + z * (pS3 + z * (pS4 + z * pS5)))));
        q = one + z * (qS1 + z * (qS2 + z * (qS3 + z * qS4)));
        r = p / q;
        w = r * s + c;
        return 2.0f * (df + w);
    }
}

// ---- glibc 2.3x atanf / atan2f (sysdeps/ieee754/flt-32/s_atanf.c, e_atan2f.c, fdlibm): float arithmetic only.
// Pinned against the host libm: atanf over all 2^32 floats, atan2f over 2*10^8 pairs (0 mismatches).
B200_HD float pt_atanf(float x) {
    const float atanhi[4] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f, 1.5707962513e+00f};
    const float atanlo[4] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f, 7.5497894159e-08f};
    const float aT0 = 3.3333334327e-01f, aT1 = -2.0000000298e-01f, aT2 = 1.4285714924e-01f, aT3 = -1.1111110449e-01f,
                aT4 = 9.0908870101e-02f, aT5 = -7.6918758452e-02f, aT6 = 6.6610731184e-02f, aT7 = -5.8335702866e-02f,
                aT8 = 4.9768779427e-02f, aT9 = -3.6531571299e-02f, aT10 = 1.6285819933e-02f;
    float w, s1, s2, z;
    const int32_t hx = (int32_t)float_as_uint(x), ix = hx & 0x7fffffff;
    int id;
    if (ix >= 0x4c000000) {
        if (ix > 0x7f800000) return x + x;
        if (hx > 0) return atanhi[3] + atanlo[3];
        return -atanhi[3] - atanlo[3];
    }
    if (ix < 0x3ee00000) {
        if (ix < 0x31000000) return x;
        id = -1;
    } else {
        x = pt_abs(x);
        if (ix < 0x3f980000) {
            if (ix < 0x3f300000) {
                id = 0;
                x = (2.0f * x - 1.0f) / (2.0f + x);
            } else {
                id = 1;
                x = (x - 1.0f) / (x + 1.0f);
            }
        } else {
            if (ix < 0x401c0000) {
                id = 2;
                x = (x - 1.5f) / (1.0f + 1.5f * x);
            } else {
                id = 3;
                x = -1.0f / x;
            }
        }
    }
    z = x * x;
    w = z * z;
    s1 = z * (aT0 + w * (aT2 + w * (aT4 + w * (aT6 + w * (aT8 + w * aT10)))));
    s2 = w * (aT1 + w * (aT3 + w * (aT5 + w * (aT7 + w * aT9))));
    if (id < 0) return x - x * (s1 + s2);
    z = atanhi[id] - ((x * (s1 + s2) - atanlo[id]) - x);
    return (hx < 0) ? -z : z;
}
B200_HD float pt_atan2f(float y, float x) {
    const float tiny = 1.0e-30f, pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f,
                pi_lo = -8.7422776573e-08f;
    float z;
    const int32_t hx = (int32_t)float_as_uint(x), hy = (int32_t)float_as_uint(y);
    const int32_t ix = hx & 0x7fffffff, iy = hy & 0x7fffffff;
    if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;
    if (hx == 0x3f800000) return pt_atanf(y);
    const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
    if (iy == 0) {
        if (m < 2) return y;
        return m == 2 ? pi + tiny : -pi - tiny;
    }
    if (ix == 0) return (hy < 0) ? -pi_o_2 - tiny : pi_o_2 + tiny;
    if (ix == 0x7f800000) {
        if (iy == 0x7f800000) {
            if (m == 0) return pi_o_4 + tiny;
            if (m == 1) return -pi_o_4 - tiny;
            if (m == 2) return 3.0f * pi_o_4 + tiny;
            return -3.0f * pi_o_4 - tiny;
        }
        if (m == 0) return 0.0f;
        if (m == 1) return -0.0f;
        return m == 2 ? pi + tiny : -pi - tiny;
    }
    if (iy == 0x7f800000) return (hy < 0) ? -pi_o_2 - tiny : pi_o_2 + tiny;
    const int32_t k = (iy - ix) >> 23;
    if (k > 60)
        z = pi_o_2 + 0.5f * pi_lo;
    else if (hx < 0 && k < -60)
        z = 0.0f;
    else
        z = pt_atanf(pt_abs(y / x));
    if (m == 0) return z;
    if (m == 1) return uint_as_float(float_as_uint(z) ^ 0x80000000u);
    if (m == 2) return pi - (z - pi_lo);
    return (z - pi_lo) - pi;
}

// ---- core/efloat.h:47-214
struct EFloat {
    float v, low, high;
};
B200_HD EFloat ef(float v, float err) {
    EFloat r;
    r.v = v;
    if (err == 0.f)
        r.low = r.high = v;
    else {
        r.low = next_float_down(v - err);
        r.high = next_float_up(v + err);
    }
    return r;
}
B200_HD EFloat ef_add(const EFloat &a, const EFloat &b) {
    EFloat r;
    r.v = a.v + b.v;
    r.low = next_float_down(a.low + b.low);
    r.high = next_float_up(a.high + b.high);
    return r;
}
B200_HD EFloat ef_sub(const EFloat &a, const EFloat &b) {
    EFloat r;
    r.v = a.v - b.v;
    r.low = next_float_down(a.low - b.high);
    r.high = next_float_up(a.high - b.low);
    return r;
}
B200_HD EFloat ef_mul(const EFloat &a, const EFloat &b) {
    EFloat r;
    r.v = a.v * b.v;
    const float p0 = a.low * b.low, p1 = a.high * b.low, p2 = a.low * b.high, p3 = a.high * b.high;
    r.low = next_float_down(pt_min(pt_min(p0, p1), pt_min(p2, p3)));
    r.high = next_float_up(pt_max(pt_max(p0, p1), pt_max(p2, p3)));
    return r;
}
B200_HD EFloat ef_div(const EFloat &a, const EFloat &b) {
    EFloat r;
    r.v = a.v / b.v;
    if (b.low < 0 && b.high > 0) {
        r.low = -pt_inf();
        r.high = pt_inf();
    } else {
        const float d0 = a.low / b.low, d1 = a.high / b.low, d2 = a.low / b.high, d3 = a.high / b.high;
        r.low = next_float_down(pt_min(pt_min(d0, d1), pt_min(d2, d3)));
        r.high = next_float_up(pt_max(pt_max(d0, d1), pt_max(d2, d3)));
    }
    return r;
}
// efloat.h:265-285
B200_HD bool ef_quadratic(const EFloat &A, const EFloat &B, const EFloat &C, EFloat *t0, EFloat *t1) {
    const double discrim = (double)B.v * (double)B.v - 4. * (double)A.v * (double)C.v;
    if (discrim < 0.) return false;
    const double rootDiscrim = sqrt(discrim);
    const EFloat frd = ef((float)rootDiscrim, (float)((double)PT_MACHINE_EPS * rootDiscrim));
    EFloat q;
    if (B.v < 0)
        q = ef_mul(ef(-.5f, 0.f), ef_sub(B, frd));
    else
        q = ef_mul(ef(-.5f, 0.f), ef_add(B, frd));
    *t0 = ef_div(q, A);
    *t1 = ef_div(C, q);
    if (t0->v > t1->v) {
        const EFloat tmp = *t0;
        *t0 = *t1;
        *t1 = tmp;
    }
    return true;
}

// ---- core/transform.h:303-351, :243-249
B200_HD V3 xform_point_err_in(const float *m, const V3 &pt, const V3 &ptError, V3 *absError) {
    const float x = pt.x, y = pt.y, z = pt.z;
    const float xp = m[0] * x + m[1] * y + m[2] * z + m[3];
    const float yp = m[4] * x + m[5] * y + m[6] * z + m[7];
    const float zp = m[8] * x + m[9] * y + m[10] * z + m[11];
    const float wp = m[12] * x + m[13] * y + m[14] * z + m[15];
    const float g3 = pt_gamma(3);
    absError->x = (g3 + 1.f) * (pt_abs(m[0]) * ptError.x + pt_abs(m[1]) * ptError.y + pt_abs(m[2]) * ptError.z) +
                  g3 * (pt_abs(m[0] * x) + pt_abs(m[1] * y) + pt_abs(m[2] * z) + pt_abs(m[3]));
    absError->y = (g3 + 1.f) * (pt_abs(m[4]) * ptError.x + pt_abs(m[5]) * ptError.y + pt_abs(m[6]) * ptError.z) +
                  g3 * (pt_abs(m[4] * x) + pt_abs(m[5] * y) + pt_abs(m[6] * z) + pt_abs(m[7]));
    absError->z = (g3 + 1.f) * (pt_abs(m[8]) * ptError.x + pt_abs(m[9]) * ptError.y + pt_abs(m[10]) * ptError.z) +
                  g3 * (pt_abs(m[8] * x) + pt_abs(m[9] * y) + pt_abs(m[10] * z) + pt_abs(m[11]));
    if (wp == 1.f) return mk(xp, yp, zp);
    const float inv = 1.f / wp;
    return mk(inv * xp, inv * yp, inv * zp);
}
B200_HD V3 xform_vector_err(const float *m, const V3 &v, V3 *absError) {
    const float g3 = pt_gamma(3);
    absError->x = g3 * (pt_abs(m[0] * v.x) + pt_abs(m[1] * v.y) + pt_abs(m[2] * v.z));
    absError->y = g3 * (pt_abs(m[4] * v.x) + pt_abs(m[5] * v.y) + pt_abs(m[6] * v.z));
    absError->z = g3 * (pt_abs(m[8] * v.x) + pt_abs(m[9] * v.y) + pt_abs(m[10] * v.z));
    return mk(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z,
              m[8] * v.x + m[9] * v.y + m[10] * v.z);
}
B200_HD V3 xform_normal(const float *mInv, const V3 &n) {
    return mk(mInv[0] * n.x + mInv[4] * n.y + mInv[8] * n.z, mInv[1] * n.x + mInv[5] * n.y + mInv[9] * n.z,
              mInv[2] * n.x + mInv[6] * n.y + mInv[10] * n.z);
}

// ---- Bounds3::IntersectP(ray, invDir, dirIsNeg) (core/geometry.h:1411-1438) on the leaf that holds the sphere in
// the host's BVHAccel: the reference reaches Sphere::Intersect(P) only through this test (bvh.cpp:676,713), and the
// sphere's own root can be off by more than the box test's slack (a shadow ray aimed at the limb of a distant
// sphere light is "hit" by Sphere::IntersectP at t < 1 - ShadowEpsilon but never enters the leaf's box before tMax).
B200_HD bool sphere_leaf_test(const DevSphere &sp, const V3 &ro, const V3 &rd, float rayTMax) {
    const float invDir[3] = {1 / rd.x, 1 / rd.y, 1 / rd.z};
    const int neg[3] = {invDir[0] < 0, invDir[1] < 0, invDir[2] < 0};
    const float g = 1 + 2 * pt_gamma(3);
    float tMin = ((neg[0] ? sp.leaf_hi[0] : sp.leaf_lo[0]) - ro.x) * invDir[0];
    float tMax = ((neg[0] ? sp.leaf_lo[0] : sp.leaf_hi[0]) - ro.x) * invDir[0];
    const float tyMin = ((neg[1] ? sp.leaf_hi[1] : sp.leaf_lo[1]) - ro.y) * invDir[1];
    float tyMax = ((neg[1] ? sp.leaf_lo[1] : sp.leaf_hi[1]) - ro.y) * invDir[1];
    tMax *= g;
    tyMax *= g;
    if (tMin > tyMax || tyMin > tMax) return false;
    if (tyMin > tMin) tMin = tyMin;
    if (tyMax < tMax) tMax = tyMax;
    const float tzMin = ((neg[2] ? sp.leaf_hi[2] : sp.leaf_lo[2]) - ro.z) * invDir[2];
    float tzMax = ((neg[2] ? sp.leaf_lo[2] : sp.leaf_hi[2]) - ro.z) * invDir[2];
    tzMax *= g;
    if (tMin > tzMax || tzMin > tMax) return false;
    if (tzMin > tMin) tMin = tzMin;
    if (tzMax < tMax) tMax = tzMax;
    return (tMin < rayTMax) && (tMax > 0);
}

// ---- Sphere::Intersect / IntersectP (sphere.cpp:49-212).  Returns false or *tHit (+ *is when is != nullptr, and the hit's
// uv and world-space dpdu / dpdv, sphere.cpp:102-120, when tg != nullptr).
B200_HD bool sphere_intersect(const DevSphere &sp, const V3 &ro, const V3 &rd, float rayTMax, float *tHit, Isect *is,
                              TexGeom *tg = nullptr) {
    const float radius = sp.radius;
    V3 oErr, dErr;
    V3 o = xform_point_err(sp.w2o, ro, &oErr);
    const V3 d = xform_vector_err(sp.w2o, rd, &dErr);
    const float lengthSquared = len2(d);
    if (lengthSquared > 0) {
        const float dt = dot(vabs(d), oErr) / lengthSquared;
        o = o + d * dt;
    }
    const EFloat ox = ef(o.x, oErr.x), oy = ef(o.y, oErr.y), oz = ef(o.z, oErr.z);
    const EFloat dx = ef(d.x, dErr.x), dy = ef(d.y, dErr.y), dz = ef(d.z, dErr.z);
    const EFloat a = ef_add(ef_add(ef_mul(dx, dx), ef_mul(dy, dy)), ef_mul(dz, dz));
    const EFloat b = ef_mul(ef(2.f, 0.f), ef_add(ef_add(ef_mul(dx, ox), ef_mul(dy, oy)), ef_mul(dz, oz)));
    const EFloat er = ef(radius, 0.f);
    const EFloat c = ef_sub(ef_add(ef_add(ef_mul(ox, ox), ef_mul(oy, oy)), ef_mul(oz, oz)), ef_mul(er, er));
    EFloat t0, t1;
    if (!ef_quadratic(a, b, c, &t0, &t1)) return false;
    if (t0.high > rayTMax || t1.low <= 0) return false;
    EFloat tShapeHit = t0;
    if (tShapeHit.low <= 0) {
        tShapeHit = t1;
        if (tShapeHit.high > rayTMax) return false;
    }
    // sphere.cpp:85-112: hit position; a clipped sphere (zmin / zmax / phimax) may fall back to the second root
    V3 pHit = o + d * tShapeHit.v;
    pHit = pHit * (radius / len(pHit));
    if (pHit.x == 0 && pHit.y == 0) pHit.x = 1e-5f * radius;
    if (sp.z_min > -radius || sp.z_max < radius || sp.phi_max < (PT_PI / 180) * 360.f) {
        float phi = pt_atan2f(pHit.y, pHit.x);
        if (phi < 0) phi += 2 * PT_PI;
        if ((sp.z_min > -radius && pHit.z < sp.z_min) || (sp.z_max < radius && pHit.z > sp.z_max) || phi > sp.phi_max) {
            if (tShapeHit.v == t1.v) return false;
            if (t1.high > rayTMax) return false;
            tShapeHit = t1;
            pHit = o + d * tShapeHit.v;
            pHit = pHit * (radius / len(pHit));
            if (pHit.x == 0 && pHit.y == 0) pHit.x = 1e-5f * radius;
            phi = pt_atan2f(pHit.y, pHit.x);
            if (phi < 0) phi += 2 * PT_PI;
            if ((sp.z_min > -radius && pHit.z < sp.z_min) || (sp.z_max < radius && pHit.z > sp.z_max) || phi > sp.phi_max)
                return false;
        }
    }
    *tHit = tShapeHit.v;
    if (!is) return true;
    const float theta = pt_acosf(pt_clamp(pHit.z / radius, -1.f, 1.f));
    const float zRadius = sqrtf(pHit.x * pHit.x + pHit.y * pHit.y);
    const float invZRadius = 1 / zRadius;
    const float cosPhi = pHit.x * invZRadius;
    const float sinPhi = pHit.y * invZRadius;
    const V3 dpdu = mk(-sp.phi_max * pHit.y, sp.phi_max * pHit.x, 0.f);
    const V3 dpdv = (sp.theta_max - sp.theta_min) * mk(pHit.z * cosPhi, pHit.z * sinPhi, -radius * pt_sinf(theta));
    const V3 pError = pt_gamma(5) * vabs(pHit);
    V3 n = normalize(cross(dpdu, dpdv));  // interaction.cpp:44-72
    if (sp.mat_flags & B200PT_TRI_FLIP) n = n * -1.f;
    const V3 wo = normalize(-d);
    is->p = xform_point_err_in(sp.o2w, pHit, pError, &is->pError);  // transform.cpp:262-297
    is->n = normalize(xform_normal(sp.w2o, n));
    is->wo = normalize(xform_vector(sp.o2w, wo));
    is->sdpdu = xform_vector(sp.o2w, dpdu);
    const V3 sn = normalize(xform_normal(sp.w2o, n));
    is->ns = (dot(sn, is->n) < 0.f) ? -sn : sn;
    if (tg) {
        float phi = pt_atan2f(pHit.y, pHit.x);
        if (phi < 0) phi += 2 * PT_PI;
        tg->u = phi / sp.phi_max;
        tg->v = (theta - sp.theta_min) / (sp.theta_max - sp.theta_min);
        tg->dpdu = xform_vector(sp.o2w, dpdu);
        tg->dpdv = xform_vector(sp.o2w, dpdv);
    }
    return true;
}

B200_HD V3 spherical_direction(float sinTheta, float cosTheta, float phi, const V3 &x, const V3 &y, const V3 &z) {
    return sinTheta * pt_cosf(phi) * x + sinTheta * pt_sinf(phi) * y + cosTheta * z;  // geometry.h:1488-1493
}

// Sphere::Sample(u, pdf), sphere.cpp:214-230
B200_HD LightSample sphere_sample_area(const DevSphere &sp, const float u[2], float *pdf) {
    const float z = 1 - 2 * u[0];  // UniformSampleSphere, sampling.cpp:98-103
    const float r = sqrtf(pt_max(0.f, 1.f - z * z));
    const float phi = 2 * PT_PI * u[1];
    V3 pObj = sp.radius * mk(r * pt_cosf(phi), r * pt_sinf(phi), z);
    pObj = mk(0.f + pObj.x, 0.f + pObj.y, 0.f + pObj.z);
    LightSample it;
    it.n = normalize(xform_normal(sp.w2o, pObj));
    if (sp.reverse_orientation) it.n = it.n * -1.f;
    pObj = pObj * (sp.radius / len(pObj));
    const V3 pObjError = pt_gamma(5) * vabs(pObj);
    it.p = xform_point_err_in(sp.o2w, pObj, pObjError, &it.pError);
    *pdf = 1 / sp.area;
    return it;
}
// Sphere::Sample(ref, u, pdf), sphere.cpp:232-290: a solid-angle density
B200_HD LightSample sphere_sample(const DevSphere &sp, const V3 &refP, const V3 &refPError, const V3 &refN,
                                  const float u[2], float *pdf) {
    const float radius = sp.radius;
    const V3 pCenter = xform_point(sp.o2w, mk(0.f, 0.f, 0.f));
    const V3 pOrigin = offset_ray_origin(refP, refPError, refN, pCenter - refP);
    if (len2(pOrigin - pCenter) <= radius * radius) {
        LightSample intr = sphere_sample_area(sp, u, pdf);
        V3 wi = intr.p - refP;
        if (len2(wi) == 0)
            *pdf = 0;
        else {
            wi = normalize(wi);
            *pdf *= len2(refP - intr.p) / absdot(intr.n, -wi);
        }
        if (pt_isinf(*pdf)) *pdf = 0.f;
        return intr;
    }
    const V3 wc = normalize(pCenter - refP);
    V3 wcX, wcY;
    coordinate_system(wc, &wcX, &wcY);
    const float sinThetaMax2 = radius * radius / len2(refP - pCenter);
    const float cosThetaMax = sqrtf(pt_max(0.f, 1 - sinThetaMax2));
    const float cosTheta = (1 - u[0]) + u[0] * cosThetaMax;
    const float sinTheta = sqrtf(pt_max(0.f, 1 - cosTheta * cosTheta));
    const float phi = u[1] * 2 * PT_PI;
    const float dc = len(refP - pCenter);
    const float ds = dc * cosTheta - sqrtf(pt_max(0.f, radius * radius - dc * dc * sinTheta * sinTheta));
    const float cosAlpha = (dc * dc + radius * radius - ds * ds) / (2 * dc * radius);
    const float sinAlpha = sqrtf(pt_max(0.f, 1 - cosAlpha * cosAlpha));
    const V3 nWorld = spherical_direction(sinAlpha, cosAlpha, phi, -wcX, -wcY, -wc);
    const V3 pWorld = pCenter + radius * nWorld;
    LightSample it;
    it.p = pWorld;
    it.pError = pt_gamma(5) * vabs(pWorld);
    it.n = nWorld;
    if (sp.reverse_orientation) it.n = it.n * -1.f;
    *pdf = 1 / (2 * PT_PI * (1 - cosThetaMax));
    return it;
}
// Sphere::Pdf(ref, wi), sphere.cpp:292-304 (+ Shape::Pdf, shape.cpp:72-87, from inside).  *nOut = the normal of the
// sphere where the ray from ref along wi meets it (needed by the caller for Le), valid when the result is > 0.
B200_HD float sphere_pdf(const DevSphere &sp, const V3 &refP, const V3 &refPError, const V3 &refN, const V3 &wi) {
    const float radius = sp.radius;
    const V3 pCenter = xform_point(sp.o2w, mk(0.f, 0.f, 0.f));
    const V3 pOrigin = offset_ray_origin(refP, refPError, refN, pCenter - refP);
    if (len2(pOrigin - pCenter) <= radius * radius) {
        const V3 ro = offset_ray_origin(refP, refPError, refN, wi);
        float tHit;
        Isect li;
        if (!sphere_intersect(sp, ro, wi, pt_inf(), &tHit, &li)) return 0.f;
        float pdf = len2(refP - li.p) / (absdot(li.n, -wi) * sp.area);
        if (pt_isinf(pdf)) pdf = 0.f;
        return pdf;
    }
    const float sinThetaMax2 = radius * radius / len2(refP - pCenter);
    const float cosThetaMax = sqrtf(pt_max(0.f, 1 - sinThetaMax2));
    return 1 / (2 * PT_PI * (1 - cosThetaMax));
}

// ---- object instances: TransformedPrimitive (core/primitive.cpp:70-98)
struct DevInstance {
    float w2i[16], i2w[16];        // WorldToInstance->m, InstanceToWorld->m
    int is_identity;               // InstanceToWorld.IsIdentity(): the hit stays as it is (primitive.cpp:93-94)
    float leaf_lo[3], leaf_hi[3];  // bounds of the host accelerator's leaf holding the instance
    float world_lo[3], world_hi[3];  // TransformedPrimitive::WorldBound()
    uint32_t node_off, tri_off;    // the object's BVH inside the scene's node / triangle arrays
    float obj_lo[3], obj_hi[3], obj_scale;  // padded object-space bounds of that BVH (TravBounds of wbvh_traverse.cuh)
};
// Transform::operator()(const Ray &) with WorldToInstance (transform.h:251-264): origin pushed to the edge of its
// error bounds, tMax shortened by the same step
B200_HD void instance_ray(const DevInstance &in, const V3 &ro, const V3 &rd, float rayTMax, V3 *o2, V3 *d2, float *tMax2) {
    V3 oError;
    V3 o = xform_point_err(in.w2i, ro, &oError);
    const V3 d = xform_vector(in.w2i, rd);
    const float lengthSquared = len2(d);
    float tMax = rayTMax;
    if (lengthSquared > 0) {
        const float dt = dot(vabs(d), oError) / lengthSquared;
        o = o + d * dt;
        tMax -= dt;
    }
    *o2 = o;
    *d2 = d;
    *tMax2 = tMax;
}
B200_HD bool instance_leaf_test(const DevInstance &in, const V3 &ro, const V3 &rd, float rayTMax) {
    DevSphere box;  // only the leaf bounds are read
    for (int a = 0; a < 3; ++a) {
        box.leaf_lo[a] = in.leaf_lo[a];
        box.leaf_hi[a] = in.leaf_hi[a];
    }
    return sphere_leaf_test(box, ro, rd, rayTMax);
}
// InstanceToWorld(SurfaceInteraction), transform.cpp:262-297 (tg: the texture lookup's dpdu / dpdv too)
B200_HD void instance_isect_to_world(const DevInstance &in, Isect *is, TexGeom *tg = nullptr) {
    if (in.is_identity) return;
    if (tg) {
        tg->dpdu = xform_vector(in.i2w, tg->dpdu);
        tg->dpdv = xform_vector(in.i2w, tg->dpdv);
    }
    Isect w = *is;
    w.p = xform_point_err_in(in.i2w, is->p, is->pError, &w.pError);
    w.n = normalize(xform_normal(in.w2i, is->n));
    w.wo = normalize(xform_vector(in.i2w, is->wo));
    w.sdpdu = xform_vector(in.i2w, is->sdpdu);
    const V3 sn = normalize(xform_normal(in.w2i, is->ns));
    w.ns = (dot(sn, w.n) < 0.f) ? -sn : sn;
    *is = w;
}

// ---- delta lights: PointLight / SpotLight / DistantLight::Sample_Li (point.cpp:43-52, spot.cpp:53-76,
// distant.cpp:49-60).  pdf is 1; *pTarget is the point the VisibilityTester aims at.
struct DeltaLight {
    int kind;  // B200PT_LIGHT_POINT / SPOT / DISTANT
    V3 position;
    Spec intensity;
    float cos_total_width, cos_falloff_start;
    const float *world_to_light;
    float two_world_radius;
};
B200_HD Spec delta_light_sample(const DeltaLight &l, const V3 &refP, V3 *wi, V3 *pTarget) {
    if (l.kind == 3) {
        *wi = l.position;
        *pTarget = refP + l.position * l.two_world_radius;
        return l.intensity;
    }
    *wi = normalize(l.position - refP);
    *pTarget = l.position;
    const float d2 = len2(l.position - refP);
    if (l.kind == 1) return l.intensity / d2;
    const V3 wl = normalize(xform_vector(l.world_to_light, -*wi));  // SpotLight::Falloff, spot.cpp:64-74
    const float cosTheta = wl.z;
    float falloff;
    if (cosTheta < l.cos_total_width)
        falloff = 0.f;
    else if (cosTheta >= l.cos_falloff_start)
        falloff = 1.f;
    else {
        const float delta = (cosTheta - l.cos_total_width) / (l.cos_falloff_start - l.cos_total_width);
        falloff = (delta * delta) * (delta * delta);
    }
    return l.intensity * falloff / d2;
}

// SpatialLightDistribution::ComputeDistribution, one (voxel, light) term (lightdistrib.cpp:196-275)
B200_HD float spatial_light_contrib(const SpatialGrid &g, int vx, int vy, int vz, const V3 &p0, const V3 &p1,
                                    const V3 &p2, bool flip, const TriShading &sh, const Spec &lemit, bool twoSided,
                                    const DevSphere *sphere, const DeltaLight *delta) {
    const int pi[3] = {vx, vy, vz};
    float lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        const float t0 = (float)pi[a] / (float)g.nv[a], t1 = (float)(pi[a] + 1) / (float)g.nv[a];
        const float b0 = lerpf(t0, g.wb_min[a], g.wb_max[a]), b1 = lerpf(t1, g.wb_min[a], g.wb_max[a]);
        lo[a] = pt_min(b0, b1);
        hi[a] = pt_max(b0, b1);
    }
    float contrib = 0.f;
    for (int i = 0; i < 128; ++i) {
        const V3 po = mk(lerpf(radical_inverse(0, i), lo[0], hi[0]), lerpf(radical_inverse(1, i), lo[1], hi[1]),
                         lerpf(radical_inverse(2, i), lo[2], hi[2]));
        const float u[2] = {radical_inverse(3, i), radical_inverse(4, i)};
        float pdf;
        LightSample ps;
        V3 w;
        if (delta) {  // Sample_Li of a delta light: pdf 1 (lightdistrib.cpp:230-236)
            V3 wiD, pT;
            const Spec LiD = delta_light_sample(*delta, po, &wiD, &pT);
            contrib += lum(LiD) / 1.f;
            continue;
        }
        if (sphere) {
            // Interaction(po, Normal3f(), Vector3f(), ...) (lightdistrib.cpp:222-223): no normal, no error bounds;
            // Sphere::Sample(ref, u, pdf) already returns a solid-angle density
            ps = sphere_sample(*sphere, po, mk(0.f, 0.f, 0.f), mk(0.f, 0.f, 0.f), u, &pdf);
            w = ps.p - po;
        } else {
            ps = triangle_sample(p0, p1, p2, flip, sh, u, &pdf);
            w = ps.p - po;
        }
        if (sphere) {
        } else if (len2(w) == 0)
            pdf = 0;
        else {
            w = normalize(w);
            pdf *= len2(po - ps.p) / absdot(ps.n, -w);
            if (pt_isinf(pdf)) pdf = 0.f;
        }
        Spec Li = rgb1(0.f);
        if (pdf == 0 || len2(ps.p - po) == 0) {
            pdf = 0;
        } else {
            const V3 wi = normalize(ps.p - po);
            Li = (twoSided || dot(ps.n, -wi) > 0) ? lemit : rgb1(0.f);
        }
        if (pdf > 0) contrib += lum(Li) / pdf;
    }
    return contrib;
}

}  // namespace B200PT_NS
#endif
