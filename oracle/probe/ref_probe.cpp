// oracle/probe/ref_probe.cpp -- TEST INFRASTRUCTURE, not product code.
//
// Harness linked against the UNMODIFIED reference (oracle/_ref/libpbrt_ref.a)
// that calls reference classes directly and prints / writes what they return.
// It is how the golden fixtures under tests/golden/ are produced
// (tests/golden/make_golden.py) and how kernel-level parity is checked against
// the real BVHAccel / Triangle / SobolSampler / PerspectiveCamera instead of
// only against the restatement in oracle/pt_oracle.cpp.
//
// Sub-commands (all output little-endian raw binary or hex-float text):
//   tables <out.bin> <ndims>      SobolMatrices32[0:ndims], VdCSobolMatrices, VdCSobolMatricesInv
//   camera ex ey ez lx ly lz ux uy uz fov xres yres
//                                 RasterToCamera and CameraToWorld of the PerspectiveCamera pbrt builds
//   sobol x0 y0 x1 y1 spp px py sample dim0 n    SobolSampler::SampleDimension stream
//   halton x0 y0 x1 y1 spp px py sample dim0 n   HaltonSampler::SampleDimension stream (first line: the index)
//   haltonperms <out.bin> <nbases>                HaltonSampler::radicalInversePermutations[0:PrimeSums[nbases]]
//   camrays <camera args> spp px py n             GetCameraSample + GenerateRayDifferential main rays
//   intersect <tris.f32> <rays.bin> <out.bin>     BVHAccel (SAH, maxnodeprims 4) Intersect + IntersectP
//   consts                                        default copper eta/k RGB, RoughnessToAlpha samples
//   mipmap <req.bin> <out.bin>                    MIPMap<RGBSpectrum | Float> built from the request's texels: the
//                                                 pyramid, weightLut, Lookup(st, dst0, dst1) and Lookup(st, width)
//   infinite <map.pfm> <req.bin> <out.bin>        InfiniteAreaLight: level 0 of Lmap, the Distribution2D tables, both
//                                                 matrices, Sample_Li, Pdf_Li and Le answers
//   differentials <req.bin> <out.bin>             SurfaceInteraction::ComputeDifferentials: dudx dvdx dudy dvdy
//   roughness <lo> <hi>                           RoughnessToAlpha of the floats with bits [lo, hi), raw to stdout
// The request and answer layouts are those of tests/texlookup.py.
// standard headers first: the access hack below must not reach them
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <iostream>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <vector>
#include <glog/logging.h>
#define private public
#define protected public
#include "accelerators/bvh.h"
#include "cameras/perspective.h"
#include "core/api.h"
#include "core/efloat.h"
#include "core/film.h"
#include "core/interaction.h"
#include "core/lowdiscrepancy.h"
#include "core/light.h"
#include "core/microfacet.h"
#include "core/mipmap.h"
#include "core/paramset.h"
#include "core/primitive.h"
#include "core/sampler.h"
#include "core/sobolmatrices.h"
#include "core/spectrum.h"
#include "core/texture.h"
#include "filters/box.h"
#include "filters/triangle.h"
#include "filters/sinc.h"
#include "filters/mitchell.h"
#include "filters/gaussian.h"
#include "lights/infinite.h"
#include "materials/matte.h"
#include "materials/metal.h"
#include "samplers/halton.h"
#include "samplers/sobol.h"
#include "shapes/sphere.h"
#include "shapes/triangle.h"
#include "textures/constant.h"
#undef private
#undef protected

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>

using namespace pbrt;

static void die(const char *m) {
    fprintf(stderr, "ref_probe: %s\n", m);
    exit(2);
}

static std::vector<float> readFloats(const char *fn) {
    FILE *f = fopen(fn, "rb");
    if (!f) die("cannot open input");
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<float> v(n / 4);
    if (fread(v.data(), 4, v.size(), f) != v.size()) die("short read");
    fclose(f);
    return v;
}

static std::vector<char> readBytes(const char *fn) {
    FILE *f = fopen(fn, "rb");
    if (!f) die("cannot open input");
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<char> v(n);
    if (n && fread(v.data(), 1, n, f) != (size_t)n) die("short read");
    fclose(f);
    return v;
}

// Reads a request field by field
struct Req {
    std::vector<char> b;
    size_t at = 0;
    template <class T>
    const T *take(size_t n) {
        if (at + n * sizeof(T) > b.size()) die("request too short");
        const T *p = (const T *)(b.data() + at);
        at += n * sizeof(T);
        return p;
    }
};

static void put(FILE *f, const void *p, size_t bytes) {
    if (bytes && fwrite(p, 1, bytes, f) != bytes) die("short write");
}

// Runs fn(i) for i in [0, n) on all cores (the reference's lookups are const)
static void parallelRange(size_t n, const std::function<void(size_t)> &fn) {
    const unsigned nt = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
    std::vector<std::thread> pool;
    const size_t per = (n + nt - 1) / nt;
    for (unsigned t = 0; t < nt; ++t) {
        const size_t lo = std::min(n, t * per), hi = std::min(n, lo + per);
        pool.emplace_back([=, &fn]() {
            for (size_t i = lo; i < hi; ++i) fn(i);
        });
    }
    for (auto &th : pool) th.join();
}

// mipmap: request int32 {channels, w, h, wrap (ImageWrap), doTrilinear, nEwa, nWidth, 0}, float maxAnisotropy, texels
// [h][w][channels], nEwa x {s, t, dst0.x, dst0.y, dst1.x, dst1.y}, nWidth x {s, t, width}.  Answer int32 {levels},
// int32 {uSize, vSize} per level, every level's texels [v][u][channels], weightLut[128], the answers (channels floats
// each).
template <typename T>
static void probeMipmap(Req &q, const int32_t *hdr, FILE *out) {
    const int ch = hdr[0], w = hdr[1], h = hdr[2], nEwa = hdr[5], nWidth = hdr[6];
    const float maxAniso = *q.take<float>(1);
    const float *tex = q.take<float>((size_t)w * h * ch);
    std::vector<T> img((size_t)w * h);
    for (size_t i = 0; i < img.size(); ++i) memcpy((void *)&img[i], tex + i * ch, sizeof(float) * ch);
    const float *ewa = q.take<float>((size_t)nEwa * 6), *wid = q.take<float>((size_t)nWidth * 3);
    MIPMap<T> mm(Point2i(w, h), img.data(), hdr[4] != 0, maxAniso, (ImageWrap)hdr[3]);
    const int32_t levels = mm.Levels();
    put(out, &levels, 4);
    for (const auto &lv : mm.pyramid) {
        const int32_t wh[2] = {lv->uSize(), lv->vSize()};
        put(out, wh, 8);
    }
    for (const auto &lv : mm.pyramid)
        for (int t = 0; t < lv->vSize(); ++t)
            for (int s = 0; s < lv->uSize(); ++s) put(out, &(*lv)(s, t), sizeof(float) * ch);
    put(out, MIPMap<T>::weightLut, sizeof(float) * 128);
    std::vector<T> a(nEwa), b(nWidth);
    parallelRange(nEwa, [&](size_t i) {
        const float *e = ewa + 6 * i;
        a[i] = mm.Lookup(Point2f(e[0], e[1]), Vector2f(e[2], e[3]), Vector2f(e[4], e[5]));
    });
    parallelRange(nWidth, [&](size_t i) { b[i] = mm.Lookup(Point2f(wid[3 * i], wid[3 * i + 1]), wid[3 * i + 2]); });
    for (const T &v : a) put(out, &v, sizeof(float) * ch);
    for (const T &v : b) put(out, &v, sizeof(float) * ch);
}

struct Cam {
    std::unique_ptr<Film> film;  // owned by camera in pbrt; keep raw here
    std::shared_ptr<PerspectiveCamera> cam;
};

static std::shared_ptr<PerspectiveCamera> makeCamera(char **a) {
    Point3f eye(atof(a[0]), atof(a[1]), atof(a[2])), look(atof(a[3]), atof(a[4]), atof(a[5]));
    Vector3f up(atof(a[6]), atof(a[7]), atof(a[8]));
    float fov = atof(a[9]);
    int xres = atoi(a[10]), yres = atoi(a[11]);
    // what pbrtLookAt + pbrtCamera do (api.cpp:993-1001, 1131-1146): curTransform = I * LookAt;
    // CameraToWorld = Inverse(curTransform)
    Transform ctm = Transform() * LookAt(eye, look, up);
    Transform *c2w = new Transform(Inverse(ctm));
    AnimatedTransform *at = new AnimatedTransform(c2w, 0, c2w, 1);
    ParamSet filmParams;
    std::unique_ptr<int[]> xr(new int[1]), yr(new int[1]);
    xr[0] = xres;
    yr[0] = yres;
    filmParams.AddInt("xresolution", std::move(xr), 1);
    filmParams.AddInt("yresolution", std::move(yr), 1);
    std::unique_ptr<std::string[]> fn(new std::string[1]);
    fn[0] = "probe.pfm";
    filmParams.AddString("filename", std::move(fn), 1);
    ParamSet empty;
    std::unique_ptr<Filter> filter(CreateBoxFilter(empty));
    Film *film = CreateFilm(filmParams, std::move(filter));
    ParamSet camParams;
    std::unique_ptr<Float[]> fv(new Float[1]);
    fv[0] = fov;
    camParams.AddFloat("fov", std::move(fv), 1);
    return std::shared_ptr<PerspectiveCamera>(CreatePerspectiveCamera(camParams, *at, film, nullptr));
}

static void printMat(const char *name, const Matrix4x4 &m) {
    printf("%s", name);
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) printf(" %a", (double)m.m[i][j]);
    printf("\n");
}

int main(int argc, char **argv) {
    if (argc < 2) die("usage: ref_probe <cmd> ...");
    std::string cmd = argv[1];
    Options opt;
    opt.nThreads = 1;
    opt.quiet = true;
    pbrtInit(opt);
    if (cmd == "tables") {
        int nd = atoi(argv[3]);
        FILE *f = fopen(argv[2], "wb");
        if (!f) die("cannot open output");
        uint32_t hdr[4] = {0x32424f53u /* "SOB2" */, (uint32_t)nd, (uint32_t)SobolMatrixSize, 26};
        fwrite(hdr, 4, 4, f);
        fwrite(SobolMatrices32, 4, (size_t)nd * SobolMatrixSize, f);
        fwrite(VdCSobolMatrices, 8, 26 * SobolMatrixSize, f);
        fwrite(VdCSobolMatricesInv, 8, 26 * SobolMatrixSize, f);
        fclose(f);
    } else if (cmd == "camera") {
        auto cam = makeCamera(argv + 2);
        printMat("raster_to_camera", cam->RasterToCamera.m);
        printMat("camera_to_world", cam->CameraToWorld.startTransform->m);
        Bounds2i sb = cam->film->GetSampleBounds();
        printf("sample_bounds %d %d %d %d\n", sb.pMin.x, sb.pMin.y, sb.pMax.x, sb.pMax.y);
        Bounds2i cb = cam->film->croppedPixelBounds;
        printf("cropped_bounds %d %d %d %d\n", cb.pMin.x, cb.pMin.y, cb.pMax.x, cb.pMax.y);
    } else if (cmd == "sobol") {
        Bounds2i sb(Point2i(atoi(argv[2]), atoi(argv[3])), Point2i(atoi(argv[4]), atoi(argv[5])));
        SobolSampler s(atoi(argv[6]), sb);
        Point2i p(atoi(argv[7]), atoi(argv[8]));
        int64_t sample = atoll(argv[9]);
        int dim0 = atoi(argv[10]), n = atoi(argv[11]);
        s.StartPixel(p);
        s.SetSampleNumber(sample);
        for (int i = 0; i < n; ++i) printf("%a\n", (double)s.SampleDimension(s.intervalSampleIndex, dim0 + i));
    } else if (cmd == "halton") {
        Bounds2i sb(Point2i(atoi(argv[2]), atoi(argv[3])), Point2i(atoi(argv[4]), atoi(argv[5])));
        HaltonSampler s(atoi(argv[6]), sb);
        Point2i p(atoi(argv[7]), atoi(argv[8]));
        int64_t sample = atoll(argv[9]);
        int dim0 = atoi(argv[10]), n = atoi(argv[11]);
        s.StartPixel(p);
        s.SetSampleNumber(sample);
        printf("%lld\n", (long long)s.intervalSampleIndex);
        for (int i = 0; i < n; ++i) printf("%a\n", (double)s.SampleDimension(s.intervalSampleIndex, dim0 + i));
    } else if (cmd == "haltonperms") {
        int nb = atoi(argv[3]);
        HaltonSampler s(1, Bounds2i(Point2i(0, 0), Point2i(16, 16)));  // the ctor fills the static table
        FILE *f = fopen(argv[2], "wb");
        if (!f) die("cannot open output");
        uint32_t count = nb < PrimeTableSize ? (uint32_t)PrimeSums[nb] : (uint32_t)HaltonSampler::radicalInversePermutations.size();
        uint32_t hdr[4] = {0x544c4148u /* "HALT" */, (uint32_t)nb, count, 0};
        fwrite(hdr, 4, 4, f);
        fwrite(HaltonSampler::radicalInversePermutations.data(), 2, count, f);
        fclose(f);
    } else if (cmd == "sphere") {
        // sphere cx cy cz radius ox oy oz dx dy dz tmax : Sphere under Translate(c): Intersect / IntersectP
        Transform o2w = Translate(Vector3f(atof(argv[2]), atof(argv[3]), atof(argv[4])));
        Transform w2o = Inverse(o2w);
        float radius = atof(argv[5]);
        Sphere sp(&o2w, &w2o, false, radius, -radius, radius, 360.f);
        Ray r(Point3f(strtof(argv[6], 0), strtof(argv[7], 0), strtof(argv[8], 0)),
              Vector3f(strtof(argv[9], 0), strtof(argv[10], 0), strtof(argv[11], 0)), strtof(argv[12], 0));
        Float tHit = 0;
        SurfaceInteraction is;
        bool hp = sp.IntersectP(r, false);
        bool h = sp.Intersect(r, &tHit, &is, false);
        printf("IntersectP %d Intersect %d t %a\n", (int)hp, (int)h, (double)tHit);
        // the EFloat roots
        Vector3f oErr, dErr;
        Ray ray = w2o(r, &oErr, &dErr);
        EFloat ox(ray.o.x, oErr.x), oy(ray.o.y, oErr.y), oz(ray.o.z, oErr.z);
        EFloat dx(ray.d.x, dErr.x), dy(ray.d.y, dErr.y), dz(ray.d.z, dErr.z);
        EFloat a = dx * dx + dy * dy + dz * dz;
        EFloat b = 2 * (dx * ox + dy * oy + dz * oz);
        EFloat c = ox * ox + oy * oy + oz * oz - EFloat(radius) * EFloat(radius);
        EFloat t0, t1;
        bool q = Quadratic(a, b, c, &t0, &t1);
        printf("o=(%a %a %a) oErr=(%a %a %a) dErr=(%a %a %a)\n", ray.o.x, ray.o.y, ray.o.z, oErr.x, oErr.y, oErr.z, dErr.x, dErr.y, dErr.z);
        printf("a=[%a %a %a] b=[%a %a %a] c=[%a %a %a]\n", a.LowerBound(), (float)a, a.UpperBound(), b.LowerBound(), (float)b,
               b.UpperBound(), c.LowerBound(), (float)c, c.UpperBound());
        printf("quadratic %d t0=[%a %a %a] t1=[%a %a %a]\n", (int)q, t0.LowerBound(), (float)t0, t0.UpperBound(), t1.LowerBound(),
               (float)t1, t1.UpperBound());
    } else if (cmd == "spheresample") {
        // spheresample cx cy cz radius  px py pz  ex ey ez  nx ny nz  u0 u1 : Sphere::Sample(ref, u, &pdf)
        Transform o2w = Translate(Vector3f(atof(argv[2]), atof(argv[3]), atof(argv[4])));
        Transform w2o = Inverse(o2w);
        float radius = atof(argv[5]);
        Sphere sp(&o2w, &w2o, false, radius, -radius, radius, 360.f);
        Interaction ref;
        ref.p = Point3f(strtof(argv[6], 0), strtof(argv[7], 0), strtof(argv[8], 0));
        ref.pError = Vector3f(strtof(argv[9], 0), strtof(argv[10], 0), strtof(argv[11], 0));
        ref.n = Normal3f(strtof(argv[12], 0), strtof(argv[13], 0), strtof(argv[14], 0));
        Point2f u(strtof(argv[15], 0), strtof(argv[16], 0));
        Float pdf = 0;
        Interaction it = sp.Sample(ref, u, &pdf);
        printf("p=(%a %a %a) n=(%a %a %a) pErr=(%a %a %a) pdf=%a\n", it.p.x, it.p.y, it.p.z, it.n.x, it.n.y, it.n.z,
               it.pError.x, it.pError.y, it.pError.z, pdf);
    } else if (cmd == "filtertable") {
        // filtertable name xwidth ywidth [p0 p1]: the Film's filterTable (film.cpp:68-77) for that PixelFilter
        std::string name = argv[2];
        ParamSet ps;
        auto addf = [&](const char *n, float v) {
            std::unique_ptr<Float[]> a(new Float[1]);
            a[0] = v;
            ps.AddFloat(n, std::move(a), 1);
        };
        addf("xwidth", atof(argv[3]));
        addf("ywidth", atof(argv[4]));
        if (name == "gaussian" && argc > 5) addf("alpha", atof(argv[5]));
        if (name == "mitchell" && argc > 6) {
            addf("B", atof(argv[5]));
            addf("C", atof(argv[6]));
        }
        if (name == "sinc" && argc > 5) addf("tau", atof(argv[5]));
        std::unique_ptr<Filter> filter;
        if (name == "box") filter.reset(CreateBoxFilter(ps));
        else if (name == "gaussian") filter.reset(CreateGaussianFilter(ps));
        else if (name == "mitchell") filter.reset(CreateMitchellFilter(ps));
        else if (name == "sinc") filter.reset(CreateSincFilter(ps));
        else if (name == "triangle") filter.reset(CreateTriangleFilter(ps));
        else die("unknown filter");
        Film film(Point2i(16, 16), Bounds2f(Point2f(0, 0), Point2f(1, 1)), std::move(filter), 35.f, "probe.pfm", 1.f);
        printf("radius %a %a\n", film.filter->radius.x, film.filter->radius.y);
        for (int i = 0; i < 256; ++i) printf("%a\n", (double)film.filterTable[i]);
        Bounds2i sb = film.GetSampleBounds();
        printf("sample_bounds_16 %d %d %d %d\n", sb.pMin.x, sb.pMin.y, sb.pMax.x, sb.pMax.y);
    } else if (cmd == "camrays") {
        auto cam = makeCamera(argv + 2);
        int spp = atoi(argv[14]);
        Point2i p(atoi(argv[15]), atoi(argv[16]));
        int n = atoi(argv[17]);
        SobolSampler s(spp, cam->film->GetSampleBounds());
        s.StartPixel(p);
        for (int i = 0; i < n; ++i) {
            s.SetSampleNumber(i);
            CameraSample cs = s.GetCameraSample(p);
            RayDifferential ray;
            cam->GenerateRayDifferential(cs, &ray);
            printf("%a %a %a %a %a %a %a\n", (double)ray.o.x, (double)ray.o.y, (double)ray.o.z, (double)ray.d.x,
                   (double)ray.d.y, (double)ray.d.z, (double)ray.tMax);
        }
    } else if (cmd == "intersect") {
        std::vector<float> tris = readFloats(argv[2]);
        std::vector<float> rays = readFloats(argv[3]);
        int nTris = (int)(tris.size() / 9);
        size_t nRays = rays.size() / 8;
        std::vector<int> idx(3 * nTris);
        for (int i = 0; i < 3 * nTris; ++i) idx[i] = i;
        Transform *identity = new Transform();
        std::vector<std::shared_ptr<Shape>> shapes =
            CreateTriangleMesh(identity, identity, false, nTris, idx.data(), 3 * nTris, (Point3f *)tris.data(),
                               nullptr, nullptr, nullptr, nullptr, nullptr);
        std::shared_ptr<Texture<Spectrum>> kd = std::make_shared<ConstantTexture<Spectrum>>(Spectrum(0.5f));
        std::shared_ptr<Texture<Float>> sig = std::make_shared<ConstantTexture<Float>>(0.f);
        std::shared_ptr<Material> mtl = std::make_shared<MatteMaterial>(kd, sig, nullptr);
        std::vector<std::shared_ptr<Primitive>> prims;
        std::map<const Primitive *, int> primIndex;
        for (int i = 0; i < nTris; ++i) {
            prims.push_back(std::make_shared<GeometricPrimitive>(shapes[i], mtl, nullptr, MediumInterface()));
            primIndex[prims.back().get()] = i;
        }
        ParamSet ps;
        std::shared_ptr<BVHAccel> bvh = CreateBVHAccelerator(prims, ps);
        FILE *f = fopen(argv[4], "wb");
        if (!f) die("cannot open output");
        for (size_t i = 0; i < nRays; ++i) {
            const float *r = &rays[8 * i];  // b200pt_ray layout: o[3], t_max, d[3], pad
            Ray ray(Point3f(r[0], r[1], r[2]), Vector3f(r[4], r[5], r[6]), r[3]);
            SurfaceInteraction isect;
            struct {
                int32_t tri;
                float t, p[3], n[3], perr[3];
                int32_t occluded;
            } out;
            memset(&out, 0, sizeof(out));
            bool hit = bvh->Intersect(ray, &isect);
            out.tri = hit ? primIndex[isect.primitive] : -1;
            if (hit) {
                out.t = ray.tMax;
                out.p[0] = isect.p.x; out.p[1] = isect.p.y; out.p[2] = isect.p.z;
                out.n[0] = isect.n.x; out.n[1] = isect.n.y; out.n[2] = isect.n.z;
                out.perr[0] = isect.pError.x; out.perr[1] = isect.pError.y; out.perr[2] = isect.pError.z;
            }
            Ray ray2(Point3f(r[0], r[1], r[2]), Vector3f(r[4], r[5], r[6]), r[3]);
            out.occluded = bvh->IntersectP(ray2) ? 1 : 0;
            fwrite(&out, sizeof(out), 1, f);
        }
        fclose(f);
    } else if (cmd == "consts") {
        ParamSet geom, mat;
        std::map<std::string, std::shared_ptr<Texture<Float>>> ft;
        std::map<std::string, std::shared_ptr<Texture<Spectrum>>> st;
        TextureParams tp(geom, mat, ft, st);
        std::unique_ptr<MetalMaterial> metal(CreateMetalMaterial(tp));
        SurfaceInteraction si;
        Spectrum eta = metal->eta->Evaluate(si), k = metal->k->Evaluate(si);
        printf("copper_eta %a %a %a\n", (double)eta[0], (double)eta[1], (double)eta[2]);
        printf("copper_k %a %a %a\n", (double)k[0], (double)k[1], (double)k[2]);
        const float rough[] = {0.f, 0.001f, 0.01f, 0.1f, 0.25f, 0.5f, 1.f};
        for (float r : rough)
            printf("roughness_to_alpha %a %a\n", (double)r,
                   (double)TrowbridgeReitzDistribution::RoughnessToAlpha(r));
    } else if (cmd == "mipmap") {
        if (argc != 4) die("usage: mipmap <req.bin> <out.bin>");
        Req q;
        q.b = readBytes(argv[2]);
        const int32_t *hdr = q.take<int32_t>(8);
        if ((hdr[0] != 1 && hdr[0] != 3) || hdr[1] < 1 || hdr[2] < 1 || hdr[3] < 0 || hdr[3] > 2) die("bad mipmap request");
        FILE *out = fopen(argv[3], "wb");
        if (!out) die("cannot open output");
        if (hdr[0] == 3)
            probeMipmap<RGBSpectrum>(q, hdr, out);
        else
            probeMipmap<Float>(q, hdr, out);
        fclose(out);
    } else if (cmd == "infinite") {
        // request: int32 {nSample, nPdf, nLe, nu, nv, 0}, float LightToWorld[16] (row major), worldRadius, ref.p[3], with nu > 0
        // an image [nv][nu] whose Distribution2D replaces the light's (sizes no map gives: the map's are powers of two),
        // nSample x u[2], nPdf x w[3], nLe x ray.d[3].  Answer: int32 {width, height, nu, nv}; level 0 of Lmap [height][width][3], every
        // pConditionalV row's func, then cdf, then funcInt; pMarginal's func, cdf, funcInt; LightToWorld.m, WorldToLight.m;
        // nSample x {wi[3], pdf, Li[3], P1().p[3]}, nPdf x Pdf_Li, nLe x Le[3]
        if (argc != 5) die("usage: infinite <map.pfm> <req.bin> <out.bin>");
        Req q;
        q.b = readBytes(argv[3]);
        const int32_t *hdr = q.take<int32_t>(6);
        const float *m = q.take<float>(16), worldRadius = *q.take<float>(1), *rp = q.take<float>(3);
        const float *img = hdr[3] > 0 ? q.take<float>((size_t)hdr[3] * hdr[4]) : nullptr;
        const float *us = q.take<float>((size_t)hdr[0] * 2), *ws = q.take<float>((size_t)hdr[1] * 3),
                    *ds = q.take<float>((size_t)hdr[2] * 3);
        Matrix4x4 mat(m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], m[8], m[9], m[10], m[11], m[12], m[13], m[14], m[15]);
        InfiniteAreaLight light(Transform(mat), Spectrum(1.f), 1, argv[2]);
        light.worldRadius = worldRadius;
        if (img) light.distribution.reset(new Distribution2D(img, hdr[3], hdr[4]));
        FILE *out = fopen(argv[4], "wb");
        if (!out) die("cannot open output");
        const auto &lv0 = *light.Lmap->pyramid[0];
        const Distribution2D &d2 = *light.distribution;
        const int32_t dims[4] = {lv0.uSize(), lv0.vSize(), d2.pConditionalV[0]->Count(), (int32_t)d2.pConditionalV.size()};
        put(out, dims, 16);
        for (int t = 0; t < lv0.vSize(); ++t)
            for (int s = 0; s < lv0.uSize(); ++s) put(out, &lv0(s, t), 12);
        for (const auto &row : d2.pConditionalV) put(out, row->func.data(), 4 * row->func.size());
        for (const auto &row : d2.pConditionalV) put(out, row->cdf.data(), 4 * row->cdf.size());
        for (const auto &row : d2.pConditionalV) put(out, &row->funcInt, 4);
        put(out, d2.pMarginal->func.data(), 4 * d2.pMarginal->func.size());
        put(out, d2.pMarginal->cdf.data(), 4 * d2.pMarginal->cdf.size());
        put(out, &d2.pMarginal->funcInt, 4);
        put(out, light.LightToWorld.m.m, 64);
        put(out, light.WorldToLight.m.m, 64);
        Interaction ref;
        ref.p = Point3f(rp[0], rp[1], rp[2]);
        std::vector<float> sa((size_t)hdr[0] * 10), pa(hdr[1]), la((size_t)hdr[2] * 3);
        parallelRange(hdr[0], [&](size_t i) {
            Vector3f wi(0, 0, 0);
            Float pdf = 0;
            VisibilityTester vis;
            const Spectrum li = light.Sample_Li(ref, Point2f(us[2 * i], us[2 * i + 1]), &wi, &pdf, &vis);
            const float o[10] = {wi.x, wi.y, wi.z, pdf, li[0], li[1], li[2], vis.p1.p.x, vis.p1.p.y, vis.p1.p.z};
            memcpy(&sa[10 * i], o, sizeof(o));
        });
        parallelRange(hdr[1], [&](size_t i) { pa[i] = light.Pdf_Li(ref, Vector3f(ws[3 * i], ws[3 * i + 1], ws[3 * i + 2])); });
        parallelRange(hdr[2], [&](size_t i) {
            RayDifferential ray(Point3f(0, 0, 0), Vector3f(ds[3 * i], ds[3 * i + 1], ds[3 * i + 2]));
            const Spectrum le = light.Le(ray);
            for (int c = 0; c < 3; ++c) la[3 * i + c] = le[c];
        });
        put(out, sa.data(), 4 * sa.size());
        put(out, pa.data(), 4 * pa.size());
        put(out, la.data(), 4 * la.size());
        fclose(out);
    } else if (cmd == "differentials") {
        // request: n x {p, n, dpdu, dpdv, rxOrigin, rxDirection, ryOrigin, ryDirection} (24 floats); answer n x {dudx, dvdx,
        // dudy, dvdy}.  n is set as given, not from dpdu x dpdv.
        if (argc != 4) die("usage: differentials <req.bin> <out.bin>");
        const std::vector<float> r = readFloats(argv[2]);
        const size_t n = r.size() / 24;
        std::vector<float> a(4 * n);
        parallelRange(n, [&](size_t i) {
            const float *c = &r[24 * i];
            SurfaceInteraction si;
            si.p = Point3f(c[0], c[1], c[2]);
            si.n = Normal3f(c[3], c[4], c[5]);
            si.dpdu = Vector3f(c[6], c[7], c[8]);
            si.dpdv = Vector3f(c[9], c[10], c[11]);
            RayDifferential ray(Point3f(0, 0, 0), Vector3f(0, 0, 1));
            ray.hasDifferentials = true;
            ray.rxOrigin = Point3f(c[12], c[13], c[14]);
            ray.rxDirection = Vector3f(c[15], c[16], c[17]);
            ray.ryOrigin = Point3f(c[18], c[19], c[20]);
            ray.ryDirection = Vector3f(c[21], c[22], c[23]);
            si.ComputeDifferentials(ray);
            const float o[4] = {si.dudx, si.dvdx, si.dudy, si.dvdy};
            memcpy(&a[4 * i], o, sizeof(o));
        });
        FILE *out = fopen(argv[3], "wb");
        if (!out) die("cannot open output");
        put(out, a.data(), 4 * a.size());
        fclose(out);
    } else if (cmd == "roughness") {
        // roughness <lo> <hi>: RoughnessToAlpha of every float with bits in [lo, hi), written to stdout in chunks
        if (argc != 4) die("usage: roughness <lo> <hi>");
        const uint64_t lo = strtoull(argv[2], 0, 0), hi = strtoull(argv[3], 0, 0);
        if (hi > (1ull << 32) || lo > hi) die("bad range");
        std::vector<float> buf(1 << 20);
        for (uint64_t s = lo; s < hi; s += buf.size()) {
            const size_t m = (size_t)std::min<uint64_t>(buf.size(), hi - s);
            for (size_t i = 0; i < m; ++i) {
                const uint32_t b = (uint32_t)(s + i);
                float x;
                memcpy(&x, &b, 4);
                buf[i] = TrowbridgeReitzDistribution::RoughnessToAlpha(x);
            }
            put(stdout, buf.data(), 4 * m);
        }
        fflush(stdout);
#ifdef B200PT_PROBE_SPECTRAL
    } else if (cmd == "spectral") {
        // spectral <out.json-ish text>: everything liboracle_spectral needs from the SampledSpectrum build:
        //   cie X|Y|Z <60 values>; rgb r g b <60 values> for every RGB triple given as r,g,b arguments (Spectrum::FromRGB,
        //   what ParamSet::AddRGBSpectrum stores, paramset.cpp:110-120); const v <60 values>; copper eta / k
        auto dump = [](const char *tag, const Spectrum &sp) {
            printf("%s", tag);
            for (int i = 0; i < nSpectralSamples; ++i) printf(" %a", (double)sp[i]);
            printf("\n");
        };
        dump("cie_x", SampledSpectrum::X);
        dump("cie_y", SampledSpectrum::Y);
        dump("cie_z", SampledSpectrum::Z);
        for (int a = 2; a + 2 < argc; a += 3) {
            Float rgb[3] = {strtof(argv[a], 0), strtof(argv[a + 1], 0), strtof(argv[a + 2], 0)};
            char tag[128];
            snprintf(tag, sizeof(tag), "rgb %a %a %a", rgb[0], rgb[1], rgb[2]);
            dump(tag, Spectrum::FromRGB(rgb));
        }
        ParamSet geom, mat;
        std::map<std::string, std::shared_ptr<Texture<Float>>> ft;
        std::map<std::string, std::shared_ptr<Texture<Spectrum>>> st;
        TextureParams tp(geom, mat, ft, st);
        std::unique_ptr<MetalMaterial> metal(CreateMetalMaterial(tp));
        SurfaceInteraction si;
        dump("copper_eta", metal->eta->Evaluate(si));
        dump("copper_k", metal->k->Evaluate(si));
#endif
    } else
        die("unknown command");
    return 0;
}
