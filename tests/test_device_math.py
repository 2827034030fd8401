"""CPU test: the device's libm restatements (pt_explog.cuh, pt_sincos.cuh, pt_sphere.cuh, pt_sincos_dbl.cuh: sampled
directions, free-flight distances and transmittances must round like the host libm the reference calls) against the host's
glibc.  tests/libm_pin.cpp checks every input of its ranges (about a minute on 8 cores; 0 mismatches, DESIGN.md
"Numerics"); this test runs every 13th input to stay quick."""
import os
import subprocess

from conftest import ROOT


def test_expf_logf_round_like_the_host_libm(tmp_path):
    exe = str(tmp_path / "libm_pin")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-builtin-sin", "-fno-builtin-cos", "-pthread",
                    os.path.join(ROOT, "tests", "libm_pin.cpp"), "-o", exe], check=True)
    r = subprocess.run([exe, "13"], capture_output=True, text=True)
    for name in ("expf", "logf", "atanf", "sinf", "cosf", "acosf", "atan2f random", "atan2f edges", "atan2f ratios",
                 "cos(double phi)", "sin(double phi)"):
        assert name + ": 0 mismatches" in r.stdout, r.stdout
    assert r.returncode == 0, r.stdout


def test_device_henyey_greenstein_passes_the_references_hg_tests(tmp_path):
    """src/tests/hg.cpp restated for the device's phase function (pt_core.cuh phase_hg / hg_sample_p, compiled for the host):
    SamplingMatch (the sampled pdf equals p(wo, wi) within 1e-4), SamplingOrientationForward / Backward (g = +-0.95),
    Normalized (the mean of p over uniform directions is 1/4pi within 1e-3)."""
    src = tmp_path / "hg.cpp"
    src.write_text(r'''
#include <cmath>
#include <cstdio>
#include <random>
#include "pt_core.cuh"
using namespace b200pt;
static std::mt19937 rng(7);
static float U() { return std::uniform_real_distribution<float>(0.f, 1.f)(rng); }
static V3 uniformSphere() {  // sampling.cpp:132-137
    float u0 = U(), u1 = U();
    float z = 1 - 2 * u0, r = std::sqrt(std::max(0.f, 1 - z * z)), phi = 2 * PT_PI * u1;
    return mk(r * std::cos(phi), r * std::sin(phi), z);
}
int main() {
    int fail = 0;
    for (float g = -.75f; g <= 0.75f; g += 0.25f)  // SamplingMatch
        for (int i = 0; i < 100; ++i) {
            V3 wo = uniformSphere(), wi;
            float u[2] = {U(), U()};
            float p0 = hg_sample_p(g, wo, &wi, u);
            if (!(std::fabs(p0 - phase_hg(dot(wo, wi), g)) <= 1e-4f)) { ++fail; printf("SamplingMatch g=%g: %g vs %g\n", g, p0, phase_hg(dot(wo, wi), g)); }
        }
    for (float g : {0.95f, -0.95f}) {  // SamplingOrientationForward / Backward
        int nForward = 0, nBackward = 0;
        for (int i = 0; i < 100; ++i) {
            V3 wi;
            float u[2] = {U(), U()};
            hg_sample_p(g, mk(-1.f, 0.f, 0.f), &wi, u);
            (wi.x > 0 ? nForward : nBackward)++;
        }
        if (g > 0 ? !(nForward >= 10 * nBackward) : !(nBackward >= 10 * nForward)) { ++fail; printf("orientation g=%g: %d / %d\n", g, nForward, nBackward); }
    }
    for (float g = -.75f; g <= 0.75f; g += 0.25f) {  // Normalized
        V3 wo = uniformSphere();
        double sum = 0;
        const int n = 100000;
        for (int i = 0; i < n; ++i) sum += phase_hg(dot(wo, uniformSphere()), g);
        if (!(std::fabs(sum / n - 1. / (4. * 3.14159265358979323846)) <= 1e-3)) { ++fail; printf("Normalized g=%g: %g\n", g, sum / n); }
    }
    printf(fail ? "HG FAILED\n" : "HG OK\n");
    return fail != 0;
}
''')
    exe = str(tmp_path / "hg")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, str(src), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "HG OK" in r.stdout, r.stdout


def test_device_bsdf_sampling_is_consistent_with_its_pdf_and_value(tmp_path):
    """In the spirit of src/tests/bsdfs.cpp (sampled directions must follow the BSDF's own Pdf) for the device's BSDF code,
    compiled for the host: for every material family the pdf and value returned by bsdf_sample_f equal bsdf_pdf / bsdf_f
    at the sampled direction (non-specular lobes); the pdf of the reflective families integrates to at most 1 over the sphere
    (microfacet normals that reflect below the horizon lose a little; pbrt-v3's MicrofacetTransmission::Pdf is not
    normalised -- the reference's own test leaves it out too -- so rough glass is only checked for consistency)."""
    src = tmp_path / "bsdf.cpp"
    src.write_text(r'''
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include "pt_core.cuh"
using namespace b200pt;
static std::mt19937 rng(11);
static float U() { return std::uniform_real_distribution<float>(0.f, 1.f)(rng); }
static V3 uniformSphere() {
    float z = 1 - 2 * U(), r = std::sqrt(std::max(0.f, 1 - z * z)), phi = 2 * PT_PI * U();
    return mk(r * std::cos(phi), r * std::sin(phi), z);
}
template <int M>
static int check(const b200pt_material &m, const char *name, double lo, double hi) {
    int fail = 0;
    for (int trial = 0; trial < 20; ++trial) {
        Isect is;
        is.n = is.ns = normalize(uniformSphere());
        V3 a, b;
        coordinate_system(is.ns, &a, &b);
        is.sdpdu = a;
        is.p = mk(0.f, 0.f, 0.f);
        is.pError = mk(0.f, 0.f, 0.f);
        Bsdf bsdf;
        make_bsdf<M>(m, nullptr, is, &bsdf);
        V3 wo = uniformSphere();
        if (dot(wo, is.n) < 0) wo = -wo;
        for (int i = 0; i < 200; ++i) {
            float u[2] = {U(), U()};
            V3 wi;
            float pdf = 0;
            int type = 0;
            Spec f = bsdf_sample_f(bsdf, wo, &wi, u, &pdf, BSDF_ALL & ~BSDF_SPECULAR, &type);
            if (pdf == 0 || is_black(f)) continue;
            float pdf2 = bsdf_pdf(bsdf, wo, wi, BSDF_ALL & ~BSDF_SPECULAR);
            Spec f2 = bsdf_f(bsdf, wo, wi, BSDF_ALL & ~BSDF_SPECULAR);
            if (!(std::fabs(pdf - pdf2) <= 2e-3f * std::max(pdf, pdf2)) || !(std::fabs(f.c[0] - f2.c[0]) <= 2e-3f * std::max(f.c[0], f2.c[0]) + 1e-6f)) {
                ++fail;
                if (fail < 4) printf("%s: pdf %g vs %g, f %g vs %g\n", name, pdf, pdf2, f.c[0], f2.c[0]);
            }
        }
        // the pdf integrates to (at most) 1 over the sphere: uniform-direction Monte Carlo estimate
        double sum = 0;
        const int n = 200000;
        for (int i = 0; i < n; ++i) sum += bsdf_pdf(bsdf, wo, uniformSphere(), BSDF_ALL & ~BSDF_SPECULAR);
        const double integral = sum / n * 4 * 3.14159265358979323846;
        if (bsdf_num_components(bsdf, BSDF_ALL & ~BSDF_SPECULAR) > 0 && !(integral > lo && integral < hi)) {
            ++fail;
            printf("%s: pdf integrates to %g\n", name, integral);
        }
    }
    return fail;
}
int main() {
    b200pt_material m;
    int fail = 0;
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_MATTE; m.kd[0] = m.kd[1] = m.kd[2] = .5f;
    fail += check<B200PT_MAT_MATTE>(m, "matte", 0.97, 1.03);
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_PLASTIC; m.kd[0] = m.kd[1] = m.kd[2] = .25f; m.ks[0] = m.ks[1] = m.ks[2] = .25f; m.alpha_x = m.alpha_y = 0.3f;
    fail += check<B200PT_MAT_PLASTIC>(m, "plastic", 0.9, 1.05);
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_METAL; m.eta[0] = .2f; m.eta[1] = .9f; m.eta[2] = 1.1f; m.k[0] = 3.9f; m.k[1] = 2.4f; m.k[2] = 2.2f; m.alpha_x = 0.25f; m.alpha_y = 0.4f;
    fail += check<B200PT_MAT_METAL>(m, "metal", 0.7, 1.05);
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_GLASS; m.variant = 1; m.ks[0] = m.ks[1] = m.ks[2] = 1.f; m.kt[0] = m.kt[1] = m.kt[2] = 1.f; m.index = 1.5f; m.alpha_x = 0.3f; m.alpha_y = 0.2f;
    fail += check<B200PT_MAT_GLASS>(m, "rough glass", 0.0, 1e9);
    printf(fail ? "BSDF FAILED (%d)\n" : "BSDF OK\n", fail);
    return fail != 0;
}
''')
    exe = str(tmp_path / "bsdf")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, str(src), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "BSDF OK" in r.stdout, r.stdout[-2000:]


def test_device_sample_discrete_passes_the_references_distribution1d_test(tmp_path):
    """Distribution1D.Discrete of src/tests/sampling.cpp:231-279 for the device's light-picking routine (sample_discrete over
    a cdf built the way Distribution1D's constructor builds it, sampling.h:57-71): same known answers, same behaviour
    around the cross-over at u = 0.25."""
    src = tmp_path / "d1d.cpp"
    src.write_text(r'''
#include <cmath>
#include <cstdio>
#include "pt_core.cuh"
using namespace b200pt;
#define EXPECT(c) do { if (!(c)) { ++fail; printf("line %d: %s\n", __LINE__, #c); } } while (0)
int main() {
    int fail = 0;
    const int n = 4;
    float func[n] = {0, 1.f, 0.f, 3.f}, cdf[n + 1];
    cdf[0] = 0;
    for (int i = 1; i < n + 1; ++i) cdf[i] = cdf[i - 1] + func[i - 1] / n;
    const float funcInt = cdf[n];
    for (int i = 1; i < n + 1; ++i) cdf[i] /= funcInt;
    float pdf;
    EXPECT(sample_discrete(cdf, func, funcInt, n, 0.f, &pdf) == 1 && pdf == 0.25f);
    EXPECT(sample_discrete(cdf, func, funcInt, n, 0.125f, &pdf) == 1 && pdf == 0.25f);
    EXPECT(sample_discrete(cdf, func, funcInt, n, .24999f, &pdf) == 1 && pdf == 0.25f);
    EXPECT(sample_discrete(cdf, func, funcInt, n, .250001f, &pdf) == 3 && pdf == 0.75f);
    EXPECT(sample_discrete(cdf, func, funcInt, n, 0.625f, &pdf) == 3 && pdf == 0.75f);
    EXPECT(sample_discrete(cdf, func, funcInt, n, PT_ONE_MINUS_EPS, &pdf) == 3 && pdf == 0.75f);
    EXPECT(sample_discrete(cdf, func, funcInt, n, 1.f, &pdf) == 3 && pdf == 0.75f);
    float u = .25f, uMax = .25f;
    for (int i = 0; i < 20; ++i) {
        u = next_float_down(u);
        uMax = next_float_up(uMax);
    }
    for (; u < uMax; u = next_float_up(u)) {
        int interval = sample_discrete(cdf, func, funcInt, n, u, &pdf);
        if (interval == 3) break;
        EXPECT(interval == 1);
    }
    EXPECT(u < uMax);
    for (; u <= uMax; u = next_float_up(u)) EXPECT(sample_discrete(cdf, func, funcInt, n, u, &pdf) == 3);
    printf(fail ? "D1D FAILED\n" : "D1D OK\n");
    return fail != 0;
}
''')
    exe = str(tmp_path / "d1d")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, str(src), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "D1D OK" in r.stdout, r.stdout


def test_device_float_utilities_pass_the_references_fp_tests(tmp_path):
    """src/tests/fp_tests.cpp for the device's versions (host-compiled): FloatingPoint.NextUpDownFloat (== std::nextafter,
    the signed-zero and infinity cases) and EFloat.Add / Sub / Mul / Div (the exact result of operands chosen anywhere inside
    -- or at the ends of -- their intervals lies inside the result's interval; the Sphere quadratic relies on it)."""
    src = tmp_path / "fp.cpp"
    src.write_text(r'''
#include <cmath>
#include <cstdio>
#include <random>
#include "pt_sphere.cuh"
using namespace b200pt;
#define EXPECT(c) do { if (!(c)) { if (++fail < 6) printf("line %d: %s\n", __LINE__, #c); } } while (0)
static std::mt19937 rng(1);
static float U() { return std::uniform_real_distribution<float>(0.f, 1.f)(rng); }
static float anyFloat() { float f; do { f = uint_as_float((uint32_t)rng()); } while (std::isnan(f)); return f; }
static EFloat getFloat() {  // fp_tests.cpp:99-137: a value with no, small, bigger or large relative error
    float minExp = -6, maxExp = 6;
    float logu = minExp + (maxExp - minExp) * U();
    float val = std::pow(10.f, logu), err = 0;
    switch (rng() % 4) {
    case 0: break;
    case 1: err = std::fabs(uint_as_float(float_as_uint(val) + rng() % 1024) - val); break;
    case 2: err = std::fabs(uint_as_float(float_as_uint(val) + rng() % (1024 * 1024)) - val); break;
    case 3: err = (4 * U()) * std::fabs(val); break;
    }
    return ef((U() < .5f ? -1.f : 1.f) * val, err);
}
static double getPrecise(const EFloat &e) {  // :141-161
    switch (rng() % 3) {
    case 0: return e.low;
    case 1: return e.high;
    default: {
        float t = U();
        double p = (1 - t) * e.low + t * e.high;
        return p > e.high ? e.high : (p < e.low ? e.low : p);
    }
    }
}
int main() {
    int fail = 0;
    const float inf = pt_inf();
    EXPECT(next_float_up(-0.f) > 0.f);
    EXPECT(next_float_down(0.f) < 0.f);
    EXPECT(next_float_up(inf) == inf);
    EXPECT(next_float_down(inf) < inf);
    EXPECT(next_float_down(-inf) == -inf);
    EXPECT(next_float_up(-inf) > -inf);
    for (int i = 0; i < 100000; ++i) {
        float f = anyFloat();
        if (std::isinf(f)) continue;
        EXPECT(std::nextafter(f, inf) == next_float_up(f));
        EXPECT(std::nextafter(f, -inf) == next_float_down(f));
    }
    for (int trial = 0; trial < 1000000; ++trial) {
        EFloat a = getFloat(), b = getFloat();
        double pa = getPrecise(a), pb = getPrecise(b);
        EFloat r = ef_add(a, b);
        float p = (float)(pa + pb);
        EXPECT(p >= r.low && p <= r.high);
        r = ef_sub(a, b);
        p = (float)(pa - pb);
        EXPECT(p >= r.low && p <= r.high);
        r = ef_mul(a, b);
        p = (float)(pa * pb);
        EXPECT(p >= r.low && p <= r.high);
        const float bErr = (b.high - b.low) / 2;  // GetAbsoluteError
        if ((double)b.low * b.high < 0. || bErr > .25 * std::fabs(b.low)) continue;
        r = ef_div(a, b);
        p = (float)(pa / pb);
        EXPECT(p >= r.low && p <= r.high);
    }
    printf(fail ? "FP FAILED (%d)\n" : "FP OK\n", fail);
    return fail != 0;
}
''')
    exe = str(tmp_path / "fp")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, str(src), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "FP OK" in r.stdout, r.stdout


def test_device_triangle_passes_the_references_reintersect_test(tmp_path):
    """Triangle.Reintersect of src/tests/shapes.cpp:152-203 for the device's triangle code (host-compiled): a ray spawned from
    an intersection -- in a random direction (SpawnRay) or towards a random point (SpawnRayTo) -- never hits the triangle it
    left, over triangles and origins whose coordinates span 10^-8 .. 10^8.  Pins fill_isect's error bounds and
    offset_ray_origin."""
    src = tmp_path / "re.cpp"
    src.write_text(r'''
#include <cmath>
#include <cstdio>
#include <random>
#include "pt_core.cuh"
using namespace b200pt;
int main() {
    long fail = 0, tested = 0;
    for (int i = 0; i < 1000; ++i) {
        std::mt19937 rng(i);
        auto U = [&]() { return std::uniform_real_distribution<float>(0.f, 1.f)(rng); };
        auto pExp = [&]() { return std::pow(10.f, -8.f + 16.f * U()); };
        V3 v[3];
        for (int j = 0; j < 3; ++j) v[j] = mk(pExp(), pExp(), pExp());
        if (len2(cross(v[1] - v[0], v[2] - v[0])) < 1e-20f) continue;
        TriShading sh;
        default_shading(&sh);
        float u[2] = {U(), U()}, pdf;
        LightSample pTri = triangle_sample(v[0], v[1], v[2], false, sh, u, &pdf);
        V3 o = mk(pExp(), pExp(), pExp());
        V3 d = pTri.p - o;
        TriHit h;
        if (!triangle_test(v[0], v[1], v[2], o, make_shear(d), pt_inf(), &h)) continue;
        Isect is;
        fill_isect(v[0], v[1], v[2], false, sh, h, d, &is);
        for (int j = 0; j < 10000; ++j) {
            float z = 1 - 2 * U(), r = std::sqrt(std::max(0.f, 1 - z * z)), phi = 2 * PT_PI * U();
            V3 w = mk(r * std::cos(phi), r * std::sin(phi), z);
            V3 ro = offset_ray_origin(is.p, is.pError, is.n, w);  // isect.SpawnRay(w)
            TriHit h2;
            ++tested;
            if (triangle_test(v[0], v[1], v[2], ro, make_shear(w), pt_inf(), &h2)) ++fail;
            V3 p2 = mk(pExp(), pExp(), pExp());
            ro = offset_ray_origin(is.p, is.pError, is.n, p2 - is.p);  // isect.SpawnRayTo(p2), interaction.h:66-71: d = p2 - p
            if (triangle_test(v[0], v[1], v[2], ro, make_shear(p2 - is.p), PT_SHADOW_TMAX, &h2)) ++fail;
        }
    }
    printf("%ld spawned ray pairs, %ld re-intersections\n%s\n", tested, fail, fail ? "REINTERSECT FAILED" : "REINTERSECT OK");
    return fail != 0;
}
''')
    exe = str(tmp_path / "re")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, str(src), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "REINTERSECT OK" in r.stdout, r.stdout


def test_device_sphere_passes_the_references_sphere_tests(tmp_path):
    """FullSphere.Reintersect, PartialSphere.Reintersect and ParialSphere.Normal of src/tests/shapes.cpp:367-497 for the
    device's Sphere code (host-compiled pt_sphere.cuh): rays spawned from a hit into the normal's hemisphere never hit the
    sphere again (radii 10^-4 .. 10^4, origins 10^-8 .. 10^8, clipped in z and phi), and the normal is radial."""
    src = tmp_path / "sph.cpp"
    src.write_text(r'''
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include "pt_sphere.cuh"
using namespace b200pt;
static DevSphere make(float radius, float zMin, float zMax, float phiMaxDeg) {
    DevSphere s;
    memset(&s, 0, sizeof(s));
    for (int i = 0; i < 4; ++i) s.o2w[5 * i] = s.w2o[5 * i] = 1.f;
    s.radius = radius;  // Sphere constructor, sphere.h:50-58
    s.z_min = pt_clamp(pt_min(zMin, zMax), -radius, radius);
    s.z_max = pt_clamp(pt_max(zMin, zMax), -radius, radius);
    s.theta_min = pt_acosf(pt_clamp(pt_min(zMin, zMax) / radius, -1.f, 1.f));
    s.theta_max = pt_acosf(pt_clamp(pt_max(zMin, zMax) / radius, -1.f, 1.f));
    s.phi_max = (PT_PI / 180) * pt_clamp(phiMaxDeg, 0.f, 360.f);
    for (int a = 0; a < 3; ++a) {  // no accelerator leaf in this test: a box that never culls
        s.leaf_lo[a] = -pt_inf();
        s.leaf_hi[a] = pt_inf();
    }
    return s;
}
int main() {
    long fail = 0, tested = 0, normals = 0;
    for (int partial = 0; partial < 2; ++partial)
        for (int i = 0; i < 100; ++i) {
            std::mt19937 rng(1000 * partial + i);
            auto U = [&]() { return std::uniform_real_distribution<float>(0.f, 1.f)(rng); };
            auto pExp = [&](float e) { return std::pow(10.f, -e + 2 * e * U()); };
            auto lerp = [](float t, float a, float b) { return (1 - t) * a + t * b; };
            const float radius = pExp(4);
            float zMin = -radius, zMax = radius, phiMax = 360;
            if (partial) {
                zMin = U() < 0.5f ? -radius : lerp(U(), -radius, radius);
                zMax = U() < 0.5f ? radius : lerp(U(), -radius, radius);
                phiMax = U() < 0.5f ? 360.f : U() * 360.f;
            }
            const DevSphere s = make(radius, zMin, zMax, phiMax);
            V3 o = mk(pExp(8), pExp(8), pExp(8));
            // destination: a random point in the sphere's bounding box (Sphere::ObjectBound, sphere.cpp:44-47)
            V3 p2 = mk(lerp(U(), -radius, radius), lerp(U(), -radius, radius), lerp(U(), s.z_min, s.z_max));
            V3 d = p2 - o;
            if (U() < .5f) d = normalize(d);
            float tHit;
            Isect is;
            if (!sphere_intersect(s, o, d, pt_inf(), &tHit, &is)) continue;
            if (partial) {  // ParialSphere.Normal: EXPECT_FLOAT_EQ(1, dot) = within 4 ulps
                const float dt = dot(normalize(is.n), normalize(is.p));
                ++normals;
                if (!(std::fabs(dt - 1.f) <= 4 * 1.1920929e-7f)) { ++fail; printf("normal: dot %a\n", dt); }
            }
            for (int j = 0; j < 10000; ++j) {
                float z = 1 - 2 * U(), r = std::sqrt(std::max(0.f, 1 - z * z)), phi = 2 * PT_PI * U();
                V3 w = mk(r * std::cos(phi), r * std::sin(phi), z);
                if (dot(w, is.n) < 0) w = -w;  // Faceforward(w, isect.n)
                V3 ro = offset_ray_origin(is.p, is.pError, is.n, w);
                float t2;
                ++tested;
                if (sphere_intersect(s, ro, w, pt_inf(), &t2, nullptr)) ++fail;
                V3 q = mk(pExp(8), pExp(8), pExp(8));
                w = q - is.p;
                if (dot(w, is.n) < 0) w = -w;
                q = is.p + w;
                ro = offset_ray_origin(is.p, is.pError, is.n, q - is.p);  // SpawnRayTo(Point3f): d = p2 - p
                if (sphere_intersect(s, ro, q - is.p, PT_SHADOW_TMAX, &t2, nullptr)) ++fail;
            }
        }
    printf("%ld spawned ray pairs, %ld normals, %ld failures\n%s\n", tested, normals, fail, fail ? "SPHERE FAILED" : "SPHERE OK");
    return fail != 0;
}
''')
    exe = str(tmp_path / "sph")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, str(src), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "SPHERE OK" in r.stdout, r.stdout[-1500:]


def test_device_radical_inverses_pass_the_references_lowdiscrepancy_tests(tmp_path):
    """LowDiscrepancy.RadicalInverse and LowDiscrepancy.ScrambledRadicalInverse of src/tests/sampling.cpp:15-74 for the device's
    Halton arithmetic (host-compiled): base 2 equals the bit reversal exactly; the permuted radical inverse in the first 128
    prime bases agrees with the naive digit loop within 1e-5 for the reference's seven indices."""
    src = tmp_path / "ld.cpp"
    src.write_text(r'''
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>
#include "pt_core.cuh"
using namespace b200pt;
int main() {
    int fail = 0;
    for (int a = 0; a < 1024; ++a)
        if (reverse_bits32((uint32_t)a) * 2.3283064365386963e-10f != radical_inverse(0, (uint64_t)a)) ++fail;
    std::vector<int> primes;
    for (int n = 2; (int)primes.size() < 128; ++n) {
        bool p = true;
        for (int q : primes) if (n % q == 0) { p = false; break; }
        if (p) primes.push_back(n);
    }
    for (int dim = 0; dim < 128; ++dim) {
        std::mt19937 rng(dim);
        const int base = primes[dim];
        std::vector<uint16_t> perm;
        for (int i = 0; i < base; ++i) perm.push_back((uint16_t)(base - 1 - i));
        std::shuffle(perm.begin(), perm.end(), rng);
        for (uint32_t index : {0u, 1u, 2u, 1151u, 32351u, 4363211u, 681122u}) {
            float val = 0, invBase = 1.f / base, invBi = invBase;
            uint32_t a = index;
            for (int i = 0; i < 32; ++i) {  // the naive loop over 32 digits, trailing perm[0] digits included
                val += perm[a % base] * invBi;
                a /= base;
                invBi *= invBase;
            }
            const float got = halton_radical_inverse((uint32_t)base, perm.data(), index);
            if (!(std::fabs(val - got) <= 1e-5f)) { if (++fail < 5) printf("base %d index %u: %g vs %g\n", base, index, val, got); }
        }
    }
    printf(fail ? "LD FAILED (%d)\n" : "LD OK\n", fail);
    return fail != 0;
}
''')
    exe = str(tmp_path / "ld")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, str(src), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "LD OK" in r.stdout, r.stdout


def test_lazy_spectra_equal_the_eager_bsdf_code_bit_for_bit(tmp_path):
    """The 60-bin shading kernel evaluates BSDF values from recipes (pt_core.cuh "Lazy spectra": FSpec / LTerm) instead of
    holding 60-float spectra.  Compiled for the host with B200PT_NSPEC=60: for every material family (smooth / rough glass
    and the mirror included, random 60-bin rows), bsdf_f_lazy / bsdf_sample_f_lazy -- with the family's lobe-kind mask and
    with the full mask -- give, bin by bin, exactly the bits of bsdf_f / bsdf_sample_f (and the same pdf, direction, sampled
    type and is_black decision); and the eager functions instantiated with the family's mask (the RGB kernels) equal the
    unmasked ones."""
    src = tmp_path / "lazy.cpp"
    src.write_text(r'''
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#define B200PT_NSPEC 60
#define B200PT_NS b200pt_s60
#include "pt_core.cuh"
using namespace b200pt_s60;
static std::mt19937 rng(23);
static float U() { return std::uniform_real_distribution<float>(0.f, 1.f)(rng); }
static V3 uniformSphere() {
    float z = 1 - 2 * U(), r = std::sqrt(std::max(0.f, 1 - z * z)), phi = 2 * PT_PI * U();
    return mk(r * std::cos(phi), r * std::sin(phi), z);
}
static int fail = 0;
template <int KINDS>
static void compare(const char *name, const Spec &f, const FSpec &l, float s) {
    bool black = true;
    for (int b0 = 0; b0 < 60; b0 += 4) {
        float v[4];
        fspec_eval4<KINDS>(l, b0, v);
        for (int j = 0; j < 4; ++j) {
            if (float_as_uint(v[j]) != float_as_uint(f.c[b0 + j])) {
                if (++fail < 6) printf("%s: bin %d lazy %a eager %a\n", name, b0 + j, v[j], f.c[b0 + j]);
            }
            if (f.c[b0 + j] * s != 0.f) black = false;
        }
    }
    if (fspec_is_black<KINDS>(l, s) != black) { ++fail; printf("%s: is_black differs\n", name); }
}
template <int M>
static void check(const b200pt_material &m, const char *name) {
    constexpr int K = mat_kinds(M);
    float rows[5 * 60];
    for (int i = 0; i < 5 * 60; ++i) rows[i] = 0.05f + 3.5f * U();
    if (M == B200PT_MAT_PLASTIC || M == B200PT_MAT_MATTE || M == B200PT_MAT_GLASS)
        for (int i = 0; i < 3 * 60; ++i) rows[i] = U();
    for (int trial = 0; trial < 40; ++trial) {
        Isect is;
        is.n = is.ns = normalize(uniformSphere());
        V3 a, b;
        coordinate_system(is.ns, &a, &b);
        is.sdpdu = a;
        is.p = is.pError = mk(0.f, 0.f, 0.f);
        Bsdf bsdf;
        make_bsdf<M>(m, rows, is, &bsdf);
        V3 wo = uniformSphere();
        for (int i = 0; i < 100; ++i) {
            const V3 wi = uniformSphere();
            for (int flags : {(int)BSDF_ALL, (int)(BSDF_ALL & ~BSDF_SPECULAR)}) {
                const Spec f = bsdf_f(bsdf, wo, wi, flags);
                // the eager code under the family's lobe-kind mask (what the RGB shading kernels instantiate) against the full mask
                const Spec fk = bsdf_f<K>(bsdf, wo, wi, flags);
                if (memcmp(&f, &fk, sizeof(Spec)) != 0 ||
                    float_as_uint(bsdf_pdf<K>(bsdf, wo, wi, flags)) != float_as_uint(bsdf_pdf(bsdf, wo, wi, flags))) {
                    if (++fail < 6) printf("%s: masked eager bsdf_f / bsdf_pdf differ from the unmasked ones\n", name);
                }
                compare<K>(name, f, bsdf_f_lazy<K>(bsdf, wo, wi, flags), absdot(wi, bsdf.ns));
                compare<KM_ALL>(name, f, bsdf_f_lazy<KM_ALL>(bsdf, wo, wi, flags), 1.f);
                float u[2] = {U(), U()};
                V3 w1 = mk(0.f, 0.f, 0.f), w2 = w1, w3 = w1;
                float p1 = 0, p2 = 0, p3 = 0;
                int t1 = 0, t2 = 0, t3 = 0;
                const Spec fs = bsdf_sample_f(bsdf, wo, &w1, u, &p1, flags, &t1);
                {
                    V3 wk = mk(0.f, 0.f, 0.f);
                    float pk = 0;
                    int tk = 0;
                    const Spec fsk = bsdf_sample_f<K>(bsdf, wo, &wk, u, &pk, flags, &tk);
                    if (memcmp(&fs, &fsk, sizeof(Spec)) != 0 || float_as_uint(pk) != float_as_uint(p1) || tk != t1 ||
                        (!is_black(fs) && memcmp(&wk, &w1, sizeof(V3)) != 0)) {
                        if (++fail < 6) printf("%s: masked eager bsdf_sample_f differs from the unmasked one\n", name);
                    }
                }
                const FSpec ls = bsdf_sample_f_lazy<K>(bsdf, wo, &w2, u, &p2, flags, &t2);
                const FSpec la = bsdf_sample_f_lazy<KM_ALL>(bsdf, wo, &w3, u, &p3, flags, &t3);
                compare<K>(name, fs, ls, 1.f);
                compare<KM_ALL>(name, fs, la, 1.f);
                const bool same = float_as_uint(p1) == float_as_uint(p2) && float_as_uint(p1) == float_as_uint(p3) && t1 == t2 && t1 == t3 &&
                                  (is_black(fs) || (memcmp(&w1, &w2, sizeof(V3)) == 0 && memcmp(&w1, &w3, sizeof(V3)) == 0));
                if (!same) { if (++fail < 6) printf("%s: sample pdf %a/%a/%a type %d/%d/%d\n", name, p1, p2, p3, t1, t2, t3); }
            }
        }
    }
}
int main() {
    b200pt_material m;
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_MATTE;
    check<B200PT_MAT_MATTE>(m, "matte");
    m.variant = 1; m.alpha_x = 0.7f; m.alpha_y = 0.4f;  // OrenNayar A, B
    check<B200PT_MAT_MATTE>(m, "oren-nayar");
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_PLASTIC; m.alpha_x = m.alpha_y = 0.3f;
    check<B200PT_MAT_PLASTIC>(m, "plastic");
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_METAL; m.alpha_x = 0.25f; m.alpha_y = 0.4f;
    check<B200PT_MAT_METAL>(m, "metal");
    memset(&m, 0, sizeof(m)); m.type = B200PT_MAT_GLASS; m.index = 1.5f;
    check<B200PT_MAT_GLASS>(m, "glass");
    m.variant = 1; m.alpha_x = 0.3f; m.alpha_y = 0.2f;
    check<B200PT_MAT_GLASS>(m, "rough glass");
    m.variant = 2;
    check<B200PT_MAT_GLASS>(m, "mirror");
    check<-1>(m, "run-time family");
    printf(fail ? "LAZY FAILED (%d)\n" : "LAZY OK\n", fail);
    return fail != 0;
}
''')
    exe = str(tmp_path / "lazy")
    inc = os.path.join(ROOT, "pbrt-v3-distributed_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I" + inc, "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe],
                   check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "LAZY OK" in r.stdout, r.stdout[-2000:]
