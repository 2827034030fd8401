// oracle/probe/alpha_probe.cpp -- TEST INFRASTRUCTURE, not product code.
//
// Linked against the UNMODIFIED reference (oracle/_ref/libpbrt_ref.a, oracle/alpha_probe.mk): builds triangle meshes
// with alpha / shadowalpha masks through the reference's own CreateTriangleMesh, ImageTexture<Float, Float> (read from
// a PFM, resampled to a power of two by MIPMap) and UVMapping2D, puts them in a BVHAccel and answers Intersect and
// IntersectP per ray.  tests/test_zz_alpha_gpu.py compares b200pt_trace_closest / b200pt_trace_any with it.
//
//   alpha_probe <request.txt> <out.bin> <levels.bin>
// request.txt, one item per line:
//   tris <file>            [n][3][3] float32, the triangles in the scene's numbering
//   uvs <file> | uvs -     [n][3][2] float32 per-vertex uvs, or none (GetUVs' defaults)
//   rays <file>            b200pt_ray records: o[3], tMax, d[3], pad
//   group <first> <count> <uv|nouv> <alpha> <shadowalpha>
//                          one mesh of triangles [first, first + count), with the uvs or without; each mask is
//                          "none - 0 0 0 0 0", "zero - 0 0 0 0 0" (ConstantTexture(0)) or
//                          "map <file.pfm> <repeat|black|clamp> <su> <sv> <du> <dv>"
// out.bin: per ray int32 triangle (-1: none), float32 ray.tMax after Intersect, int32 IntersectP
// levels.bin: per "map" mask in request order: int32 width, height, then level 0 of its MIPMap, float32 [h][w]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>
#include <string>
#include <vector>
// the MIPMap's pyramid is private
#define private public
#define protected public
#include "accelerators/bvh.h"
#include "core/api.h"
#include "core/mipmap.h"
#include "core/paramset.h"
#include "core/primitive.h"
#include "core/texture.h"
#include "shapes/triangle.h"
#include "textures/constant.h"
#include "textures/imagemap.h"
#undef private
#undef protected

using namespace pbrt;

static void die(const char *m) {
    fprintf(stderr, "alpha_probe: %s\n", m);
    exit(1);
}
static std::vector<float> readFloats(const std::string &path) {
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) die("cannot open input");
    std::vector<float> v;
    float x;
    while (fread(&x, 4, 1, f) == 1) v.push_back(x);
    fclose(f);
    return v;
}

int main(int argc, char **argv) {
    if (argc != 4) die("usage: alpha_probe <request.txt> <out.bin> <levels.bin>");
    Options opts;
    opts.quiet = true;
    pbrtInit(opts);
    std::ifstream req(argv[1]);
    std::string line;
    std::vector<float> tris, uvs, rays;
    FILE *lv = fopen(argv[3], "wb");
    if (!lv) die("cannot open levels output");
    Transform *identity = new Transform();
    std::vector<std::shared_ptr<Primitive>> prims;
    std::map<const Primitive *, int> primIndex;
    auto mask = [&](std::istringstream &in) -> std::shared_ptr<Texture<Float>> {
        std::string kind, file, wrap;
        float su, sv, du, dv;
        in >> kind >> file >> wrap >> su >> sv >> du >> dv;
        if (kind == "none") return nullptr;
        if (kind == "zero") return std::make_shared<ConstantTexture<Float>>(0.f);
        if (kind != "map") die("unknown mask kind");
        ImageWrap wm = wrap == "black" ? ImageWrap::Black : wrap == "clamp" ? ImageWrap::Clamp : ImageWrap::Repeat;
        std::unique_ptr<TextureMapping2D> map(new UVMapping2D(su, sv, du, dv));
        auto t = std::make_shared<ImageTexture<Float, Float>>(std::move(map), file, false, 8.f, wm, 1.f, false);
        const auto &l0 = *t->mipmap->pyramid[0];
        const int32_t wh[2] = {l0.uSize(), l0.vSize()};
        fwrite(wh, 4, 2, lv);
        for (int y = 0; y < wh[1]; ++y)
            for (int x = 0; x < wh[0]; ++x) {
                const float v = l0(x, y);
                fwrite(&v, 4, 1, lv);
            }
        return t;
    };
    while (std::getline(req, line)) {
        std::istringstream in(line);
        std::string key;
        in >> key;
        if (key == "tris") {
            std::string f;
            in >> f;
            tris = readFloats(f);
        } else if (key == "uvs") {
            std::string f;
            in >> f;
            if (f != "-") uvs = readFloats(f);
        } else if (key == "rays") {
            std::string f;
            in >> f;
            rays = readFloats(f);
        } else if (key == "group") {
            int first, count;
            std::string uv;
            in >> first >> count >> uv;
            std::shared_ptr<Texture<Float>> alpha = mask(in), shadow = mask(in);
            std::vector<int> idx(3 * count);
            for (int i = 0; i < 3 * count; ++i) idx[i] = i;
            std::vector<std::shared_ptr<Shape>> shapes = CreateTriangleMesh(
                identity, identity, false, count, idx.data(), 3 * count, (const Point3f *)&tris[(size_t)first * 9], nullptr,
                nullptr, uv != "uv" ? nullptr : (const Point2f *)&uvs[(size_t)first * 6], alpha, shadow);
            for (int i = 0; i < count; ++i) {
                prims.push_back(std::make_shared<GeometricPrimitive>(shapes[i], nullptr, nullptr, MediumInterface()));
                primIndex[prims.back().get()] = first + i;
            }
        }
    }
    fclose(lv);
    ParamSet ps;
    std::shared_ptr<BVHAccel> bvh = CreateBVHAccelerator(prims, ps);
    FILE *f = fopen(argv[2], "wb");
    if (!f) die("cannot open output");
    for (size_t i = 0; i + 8 <= rays.size(); i += 8) {
        const float *r = &rays[i];
        Ray ray(Point3f(r[0], r[1], r[2]), Vector3f(r[4], r[5], r[6]), r[3]);
        SurfaceInteraction isect;
        struct {
            int32_t tri;
            float t;
            int32_t occluded;
        } out;
        const bool hit = bvh->Intersect(ray, &isect);
        out.tri = hit ? primIndex[isect.primitive] : -1;
        out.t = hit ? ray.tMax : 0.f;
        Ray ray2(Point3f(r[0], r[1], r[2]), Vector3f(r[4], r[5], r[6]), r[3]);
        out.occluded = bvh->IntersectP(ray2) ? 1 : 0;
        fwrite(&out, sizeof(out), 1, f);
    }
    fclose(f);
    pbrtCleanup();
    return 0;
}
