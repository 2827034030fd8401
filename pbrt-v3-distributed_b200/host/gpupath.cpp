// gpupath.cpp -- host side of the drop-in: a pbrt Integrator that renders on
// the H100 through the C ABI (include/b200pt.h).
//
//   template <class Base> class GpuIntegrator : public Base   (Base = PathIntegrator, integrators/path.h:48-66,
//                                                          or VolPathIntegrator, integrators/volpath.h:49-66)
//       void Render(const Scene &) override               (core/integrator.h:53-58, replaces
//                                                          SamplerIntegrator::Render, integrator.cpp:228-339)
//   PathIntegrator *CreatePathIntegrator(const ParamSet&, shared_ptr<Sampler>, shared_ptr<const Camera>)
//                                                         (integrators/path.cpp:190-213; same signature, same
//                                                          parameters: maxdepth, pixelbounds, rrthreshold,
//                                                          lightsamplestrategy)
//
// pbrt has no plugin ABI: integrators are chosen by name in
// RenderOptions::MakeIntegrator (core/api.cpp:1686-1687).  This translation
// unit DEFINES pbrt::CreatePathIntegrator, so linking it in place of the
// reference's definition makes every `Integrator "path"` of an unmodified
// .pbrt file render on the GPU while parser, scene construction, Film and image
// output stay the reference's own code (see INTEGRATION.md for the link recipe
// and for the in-tree alternative of adding a "gpupath" branch to api.cpp).
//
// Render() flattens the already-built Scene into the POD descriptors of the C
// ABI.  The reference keeps the needed members private (Scene::aggregate,
// BVHAccel::primitives, GeometricPrimitive::shape/material/areaLight,
// Triangle::mesh/v, the materials' textures, Film::pixels ...); an in-tree
// integration would add `template <class> friend class GpuIntegrator;` to those classes.
// Out of tree, this file widens access for its own includes only -- it reads
// those members, never changes layout or behaviour.
//
// Error conventions follow the reference: unsupported scene features call
// Error() (core/error.h:54) and return without rendering, like a failed
// factory in pbrtWorldEnd (api.cpp:1623); there is NO CPU fallback.
#include <algorithm>
#include <chrono>
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
#include <type_traits>
#include <unordered_map>
#include <vector>
#include <glog/logging.h>

#define private public
#define protected public
#include "accelerators/bvh.h"
#include "cameras/perspective.h"
#include "core/film.h"
#include "core/integrator.h"
#include "integrators/volpath.h"
#include "media/homogeneous.h"
#include "core/light.h"
#include "core/paramset.h"
#include "core/primitive.h"
#include "core/progressreporter.h"
#include "core/sampler.h"
#include "core/scene.h"
#include "core/sobolmatrices.h"
#include "core/stats.h"
#include "core/texture.h"
#include "filters/box.h"
#include "integrators/path.h"
#include "lights/diffuse.h"
#include "lights/spot.h"
#include "lights/point.h"
#include "lights/distant.h"
#include "lights/infinite.h"
#include "materials/glass.h"
#include "materials/matte.h"
#include "materials/metal.h"
#include "materials/mirror.h"
#include "materials/plastic.h"
#include "samplers/halton.h"
#include "samplers/sobol.h"
#include "shapes/sphere.h"
#include "shapes/triangle.h"
#include "textures/constant.h"
#include "textures/imagemap.h"
#undef private
#undef protected

#include "../../include/b200pt.h"

namespace pbrt {
// Layout of BVHAccel's flattened nodes: the reference defines this struct inside accelerators/bvh.cpp:95-104 (the
// header only forward-declares it), so a host that reads the tree has to restate the 32-byte record.
struct LinearBVHNode {
    Bounds3f bounds;
    union {
        int primitivesOffset;   // leaf
        int secondChildOffset;  // interior
    };
    uint16_t nPrimitives;  // 0 -> interior node
    uint8_t axis;
    uint8_t pad[1];
};
static_assert(sizeof(LinearBVHNode) == 32, "LinearBVHNode layout");
}  // namespace pbrt

namespace pbrt {

STAT_COUNTER("Integrator/Camera rays traced (GPU)", nGpuCameraRays);
STAT_COUNTER("Intersections/Regular ray intersection tests (GPU)", nGpuRegular);
STAT_COUNTER("Intersections/Shadow ray intersection tests (GPU)", nGpuShadow);

namespace {

template <typename T>
bool ConstantValue(const std::shared_ptr<Texture<T>> &tex, T *out) {
    auto c = dynamic_cast<const ConstantTexture<T> *>(tex.get());
    if (!c) return false;
    *out = c->value;
    return true;
}

// A host built with `typedef SampledSpectrum Spectrum` (core/pbrt.h:124-125) also hands over the 60 bins of every
// spectrum (b200pt_scene_desc::material_spectra / light_spectra) and its SampledSpectrum::X / Y / Z; the library then
// computes per bin like that build does and the RGB triples are informational.
constexpr bool kSampledHost = Spectrum::nSamples != 3;
static_assert(!kSampledHost || Spectrum::nSamples == B200PT_SPECTRUM_SAMPLES, "SampledSpectrum with another bin count");

void ToRGB(const Spectrum &s, float out[3], float *bins = nullptr) {
    Float rgb[3];
    s.ToRGB(rgb);
    out[0] = rgb[0];
    out[1] = rgb[1];
    out[2] = rgb[2];
    if (kSampledHost && bins)
        for (int i = 0; i < Spectrum::nSamples; ++i) bins[i] = s[i];
}
// one light's spectrum appended to Flattened::lightSpectra
void ToRGB(const Spectrum &s, float out[3], std::vector<float> *lightSpectra) {
    ToRGB(s, out);
    if (kSampledHost)
        for (int i = 0; i < Spectrum::nSamples; ++i) lightSpectra->push_back(s[i]);
}

struct Flattened {
    std::vector<float> vertices, normals, uvs;
    std::vector<uint8_t> vertexFlags;
    bool anyNormals = false, anyUVs = false;
    std::vector<int32_t> materialId, lightId;
    std::vector<uint8_t> flip;
    std::vector<b200pt_material> materials;
    std::vector<b200pt_area_light> lights;
    std::vector<b200pt_sphere> spheres;
    std::vector<b200pt_instance> instances;
    int64_t nTopLevel = 0;
    std::vector<float> materialSpectra, lightSpectra;  // SampledSpectrum hosts: [material][5][60], [light][60]
    // VolPathIntegrator: spheres without a material whose MediumInterface is a transition (clouds): per sphere the index
    // into boundedMedia (the medium inside) or -1; boundaryOutside[k] is what the scene declares outside boundary medium k
    std::vector<int32_t> sphereMedium;
    std::vector<const Medium *> boundedMedia, boundaryOutside;
    // InfiniteAreaLights: what b200pt_scene_set_infinite_light takes, copied from the light's own members
    struct Infinite {
        int light;
        int width, height, nu, nv;
        std::vector<float> texels, condFunc, condCdf, condFuncInt, margFunc, margCdf;
        float margFuncInt, lightToWorld[16], powerRGB[3];
    };
    std::vector<Infinite> infinite;
    // ImageTextures (b200pt_scene_add_mipmap / b200pt_scene_bind_texture): every distinct MIPMap once (ImageTexture's
    // cache shares one between textures with equal TexInfo), copied from the host's pyramid, and the bound slots
    struct Mip {
        int channels, wrap, trilinear;
        float maxAniso, weightLut[128];
        std::vector<int> w, h;
        std::vector<std::vector<float>> levels;
    };
    std::vector<Mip> mipmaps;
    std::unordered_map<const void *, int> mipOf;
    struct Bind {
        int material, slot, mip;
        float su, sv, du, dv;
        int remap;
    };
    std::vector<Bind> binds;
    // alpha / shadowalpha masks (b200pt_scene_add_alpha_mask / b200pt_scene_set_alpha_masks): every distinct mask
    // texture once (w == 0: ConstantTexture(0)), and per triangle its masks or -1
    struct Alpha {
        int w, h, wrap;
        float su, sv, du, dv;
        std::vector<float> texels;
    };
    std::vector<Alpha> alphaMasks;
    std::unordered_map<const void *, int> alphaOf;
    std::vector<int32_t> alphaId, shadowAlphaId;
};

// The MIPMap of an ImageTexture as the host built it (mipmap.h:116-218): the levels, the wrap mode, the filter settings
// and weightLut, nothing recomputed
template <typename Tm>
int AddMipmap(const MIPMap<Tm> *mm, Flattened *f) {
    auto it = f->mipOf.find(mm);
    if (it != f->mipOf.end()) return it->second;
    Flattened::Mip m;
    m.channels = std::is_same<Tm, Float>::value ? 1 : 3;
    m.wrap = mm->wrapMode == ImageWrap::Repeat ? B200PT_WRAP_REPEAT : mm->wrapMode == ImageWrap::Black ? B200PT_WRAP_BLACK : B200PT_WRAP_CLAMP;
    m.trilinear = mm->doTrilinear ? 1 : 0;
    m.maxAniso = mm->maxAnisotropy;
    for (int i = 0; i < 128; ++i) m.weightLut[i] = MIPMap<Tm>::weightLut[i];
    for (const auto &lv : mm->pyramid) {
        m.w.push_back(lv->uSize());
        m.h.push_back(lv->vSize());
        std::vector<float> t;
        t.reserve((size_t)lv->uSize() * lv->vSize() * m.channels);
        for (int y = 0; y < lv->vSize(); ++y)
            for (int x = 0; x < lv->uSize(); ++x) {
                const Tm &v = (*lv)(x, y);
                for (int c = 0; c < m.channels; ++c) t.push_back(((const Float *)&v)[c]);
            }
        m.levels.push_back(std::move(t));
    }
    const int id = (int)f->mipmaps.size();
    f->mipmaps.push_back(std::move(m));
    f->mipOf[mm] = id;
    return id;
}

// A material parameter: a constant (*value) or, on RGBSpectrum hosts, an ImageTexture under UVMapping2D bound to
// (material, slot) with the given remap flag
template <typename T, typename Tm>
bool TexturedParam(const std::shared_ptr<Texture<T>> &tex, T *value, int material, int slot, int remap, Flattened *f, std::string *why) {
    if (ConstantValue(tex, value)) return true;
    auto it = dynamic_cast<const ImageTexture<Tm, T> *>(tex.get());
    if (!it) return *why = "textures other than \"constant\" and \"imagemap\"", false;
    if (kSampledHost) return *why = "image textures in a SampledSpectrum build", false;
    auto uv = dynamic_cast<const UVMapping2D *>(it->mapping.get());
    if (!uv) return *why = "imagemap textures with a mapping other than \"uv\"", false;
    *value = T(0.f);
    f->binds.push_back({material, slot, AddMipmap(it->mipmap, f), uv->su, uv->sv, uv->du, uv->dv, remap});
    return true;
}
// A mesh's alphaMask or shadowAlphaMask (triangle.cpp:718-743): *id = -1 for none, else the mask.  Inside
// Triangle::Intersect / IntersectP the texture is evaluated without differentials, so an ImageTexture<Float, Float> under
// UVMapping2D reads level 0 of its MIPMap only (copied, nothing recomputed).  A constant that is not 0 never rejects a
// hit; IntersectP's rejection of masked triangles with a zero geometric normal needs no mask either, since such
// triangles never enter the device's trees.
bool AlphaMask(const std::shared_ptr<Texture<Float>> &tex, Flattened *f, int32_t *id, std::string *why) {
    *id = -1;
    if (!tex) return true;
    auto found = f->alphaOf.find(tex.get());
    if (found != f->alphaOf.end()) return *id = found->second, true;
    Flattened::Alpha a;
    a.w = a.h = 0;
    a.wrap = B200PT_WRAP_REPEAT;
    a.su = a.sv = 1.f;
    a.du = a.dv = 0.f;
    Float c;
    if (ConstantValue(tex, &c)) {
        if (c != 0) return true;
    } else {
        auto it = dynamic_cast<const ImageTexture<Float, Float> *>(tex.get());
        if (!it) return *why = "alpha masks other than \"constant\" and \"imagemap\" textures", false;
        auto uv = dynamic_cast<const UVMapping2D *>(it->mapping.get());
        if (!uv) return *why = "alpha masks with a mapping other than \"uv\"", false;
        const MIPMap<Float> *mm = it->mipmap;
        const auto &lv = *mm->pyramid[0];
        a.w = lv.uSize();
        a.h = lv.vSize();
        a.wrap = mm->wrapMode == ImageWrap::Repeat ? B200PT_WRAP_REPEAT : mm->wrapMode == ImageWrap::Black ? B200PT_WRAP_BLACK : B200PT_WRAP_CLAMP;
        a.su = uv->su;
        a.sv = uv->sv;
        a.du = uv->du;
        a.dv = uv->dv;
        a.texels.reserve((size_t)a.w * a.h);
        for (int y = 0; y < a.h; ++y)
            for (int x = 0; x < a.w; ++x) a.texels.push_back(lv(x, y));
    }
    *id = (int32_t)f->alphaMasks.size();
    f->alphaMasks.push_back(std::move(a));
    f->alphaOf[tex.get()] = *id;
    return true;
}

bool SpectrumParam(const std::shared_ptr<Texture<Spectrum>> &tex, Spectrum *value, int material, int slot, Flattened *f, std::string *why) {
    return TexturedParam<Spectrum, RGBSpectrum>(tex, value, material, slot, 0, f, why);
}
bool FloatParam(const std::shared_ptr<Texture<Float>> &tex, Float *value, int material, int slot, bool remap, Flattened *f, std::string *why) {
    return TexturedParam<Float, Float>(tex, value, material, slot, remap ? 1 : 0, f, why);
}

// materials/{matte,plastic,metal,glass}.cpp ComputeScatteringFunctions with constant textures, or image textures the device
// evaluates per hit (material index `mi`, bindings appended to f->binds; their constants here are 0 and ignored)
// `rows`: the material's B200PT_MATERIAL_SPECTRA x 60 block (kd, ks, kt, eta, k), zero-initialised by the caller
bool ConvertMaterial(const Material *m, b200pt_material *out, float *rows, int mi, Flattened *f, std::string *why) {
    memset(out, 0, sizeof(*out));
    float *rowKd = rows, *rowKs = rows + B200PT_SPECTRUM_SAMPLES, *rowKt = rows + 2 * B200PT_SPECTRUM_SAMPLES,
          *rowEta = rows + 3 * B200PT_SPECTRUM_SAMPLES, *rowK = rows + 4 * B200PT_SPECTRUM_SAMPLES;
    Spectrum sv;
    Float fv;
    if (auto mm = dynamic_cast<const MatteMaterial *>(m)) {
        if (mm->bumpMap) return *why = "bump maps", false;
        if (!SpectrumParam(mm->Kd, &sv, mi, B200PT_TEX_KD, f, why)) return false;
        if (!ConstantValue(mm->sigma, &fv)) return *why = "a textured matte \"sigma\"", false;
        out->type = B200PT_MAT_MATTE;
        ToRGB(sv.Clamp(), out->kd, rowKd);
        if (Clamp(fv, 0, 90) != 0) {  // OrenNayar(r, sig), matte.cpp:59
            out->variant = 1;
            b200pt_host_oren_nayar(fv, &out->alpha_x, &out->alpha_y);
        }
        return true;
    }
    if (auto pm = dynamic_cast<const PlasticMaterial *>(m)) {
        if (pm->bumpMap) return *why = "bump maps", false;
        Spectrum kd, ks;
        if (!SpectrumParam(pm->Kd, &kd, mi, B200PT_TEX_KD, f, why) || !SpectrumParam(pm->Ks, &ks, mi, B200PT_TEX_KS, f, why) ||
            !FloatParam(pm->roughness, &fv, mi, B200PT_TEX_ROUGHNESS_U, pm->remapRoughness, f, why))
            return false;
        out->type = B200PT_MAT_PLASTIC;
        ToRGB(kd.Clamp(), out->kd, rowKd);
        ToRGB(ks.Clamp(), out->ks, rowKs);
        Float rough = fv;
        if (pm->remapRoughness) rough = TrowbridgeReitzDistribution::RoughnessToAlpha(rough);
        out->alpha_x = out->alpha_y = rough;
        return true;
    }
    if (auto me = dynamic_cast<const MetalMaterial *>(m)) {
        if (me->bumpMap) return *why = "bump maps", false;
        Spectrum eta, k;
        Float ur, vr;
        if (!SpectrumParam(me->eta, &eta, mi, B200PT_TEX_ETA, f, why) || !SpectrumParam(me->k, &k, mi, B200PT_TEX_K, f, why))
            return false;
        if (!FloatParam(me->uRoughness ? me->uRoughness : me->roughness, &ur, mi, B200PT_TEX_ROUGHNESS_U, me->remapRoughness, f, why) ||
            !FloatParam(me->vRoughness ? me->vRoughness : me->roughness, &vr, mi, B200PT_TEX_ROUGHNESS_V, me->remapRoughness, f, why))
            return false;
        if (me->remapRoughness) {
            ur = TrowbridgeReitzDistribution::RoughnessToAlpha(ur);
            vr = TrowbridgeReitzDistribution::RoughnessToAlpha(vr);
        }
        out->type = B200PT_MAT_METAL;
        ToRGB(eta, out->eta, rowEta);
        ToRGB(k, out->k, rowK);
        out->alpha_x = ur;
        out->alpha_y = vr;
        return true;
    }
    if (auto gm = dynamic_cast<const GlassMaterial *>(m)) {
        if (gm->bumpMap) return *why = "bump maps", false;
        Spectrum R, T;
        Float ur, vr, index;
        if (!SpectrumParam(gm->Kr, &R, mi, B200PT_TEX_KS, f, why) || !SpectrumParam(gm->Kt, &T, mi, B200PT_TEX_KT, f, why)) return false;
        if (!ConstantValue(gm->uRoughness, &ur) || !ConstantValue(gm->vRoughness, &vr))
            return *why = "a textured glass roughness", false;
        if (!ConstantValue(gm->index, &index)) return *why = "a textured glass \"index\"", false;
        out->type = B200PT_MAT_GLASS;
        ToRGB(R.Clamp(), out->ks, rowKs);
        ToRGB(T.Clamp(), out->kt, rowKt);
        out->index = index;
        if (ur != 0 || vr != 0) {  // glass.cpp:65-90
            out->variant = 1;
            if (gm->remapRoughness) {
                ur = TrowbridgeReitzDistribution::RoughnessToAlpha(ur);
                vr = TrowbridgeReitzDistribution::RoughnessToAlpha(vr);
            }
            out->alpha_x = ur;
            out->alpha_y = vr;
        }
        return true;
    }
    if (auto mr = dynamic_cast<const MirrorMaterial *>(m)) {
        if (mr->bumpMap) return *why = "bump maps", false;
        if (!SpectrumParam(mr->Kr, &sv, mi, B200PT_TEX_KS, f, why)) return false;
        out->type = B200PT_MAT_GLASS;  // the specular family; variant 2 = SpecularReflection(Kr, FresnelNoOp), mirror.cpp:45-56
        out->variant = 2;
        ToRGB(sv.Clamp(), out->ks, rowKs);
        out->index = 1.f;
        return true;
    }
    *why = "a material other than matte / plastic / metal / glass / mirror";
    return false;
}

// `volumetric`: VolPathIntegrator looks at the primitives' MediumInterfaces; of the surfaces that separate two media only
// spheres without a material are supported (the path steps over them, volpath.cpp:115-121)
bool FlattenScene(const Scene &scene, Flattened *f, std::string *why, bool volumetric) {
    auto bvh = dynamic_cast<const BVHAccel *>(scene.aggregate.get());
    if (!bvh) return *why = "an aggregate other than BVHAccel", false;
    // BVHAccel reorders its vector (orderedPrims, bvh.cpp:208); any order works as long as it is
    // used consistently -- triangle ids only name primitives
    const auto &prims = bvh->primitives;
    std::unordered_map<const Material *, int> matIndex;
    std::unordered_map<const Shape *, int> triOfShape, sphereOfShape;
    auto noTransition = [&](const GeometricPrimitive *gp) {
        if (volumetric && gp->mediumInterface.IsMediumTransition())
            return *why = "surfaces that separate two media (MediumInterface with different inside / outside)", false;
        return true;
    };
    auto materialOf = [&](const Material *m, int *id) {
        if (!m) return *why = "primitives without a material (medium boundaries)", false;
        auto it = matIndex.find(m);
        if (it == matIndex.end()) {
            b200pt_material bm;
            std::vector<float> rows((size_t)B200PT_MATERIAL_SPECTRA * B200PT_SPECTRUM_SAMPLES, 0.f);
            if (!ConvertMaterial(m, &bm, rows.data(), (int)f->materials.size(), f, why)) return false;
            it = matIndex.emplace(m, (int)f->materials.size()).first;
            f->materials.push_back(bm);
            if (kSampledHost) f->materialSpectra.insert(f->materialSpectra.end(), rows.begin(), rows.end());
        }
        *id = it->second;
        return true;
    };
    auto appendTriangle = [&](const GeometricPrimitive *gp) {
        auto tri = dynamic_cast<const Triangle *>(gp->shape.get());
        if (!tri) return *why = "a shape other than Triangle and Sphere", false;
        if (!volumetric && (gp->mediumInterface.inside || gp->mediumInterface.outside)) return *why = "participating media", false;
        if (!noTransition(gp)) return false;
        const TriangleMesh &mesh = *tri->mesh;
        if (mesh.s) return *why = "meshes with per-vertex tangents", false;
        int32_t alpha, shadowAlpha;
        if (!AlphaMask(mesh.alphaMask, f, &alpha, why) || !AlphaMask(mesh.shadowAlphaMask, f, &shadowAlpha, why)) return false;
        f->alphaId.push_back(alpha);
        f->shadowAlphaId.push_back(shadowAlpha);
        for (int v = 0; v < 3; ++v) {
            const Point3f &p = mesh.p[tri->v[v]];
            f->vertices.push_back(p.x);
            f->vertices.push_back(p.y);
            f->vertices.push_back(p.z);
            Normal3f n = mesh.n ? mesh.n[tri->v[v]] : Normal3f(0, 0, 0);
            f->normals.push_back(n.x);
            f->normals.push_back(n.y);
            f->normals.push_back(n.z);
            Point2f uv = mesh.uv ? mesh.uv[tri->v[v]] : Point2f(0, 0);
            f->uvs.push_back(uv.x);
            f->uvs.push_back(uv.y);
        }
        f->vertexFlags.push_back((mesh.n ? 1 : 0) | (mesh.uv ? 2 : 0));
        f->anyNormals |= mesh.n != nullptr;
        f->anyUVs |= mesh.uv != nullptr;
        f->flip.push_back((tri->reverseOrientation ^ tri->transformSwapsHandedness) ? 1 : 0);
        int mid;
        if (!materialOf(gp->material.get(), &mid)) return false;
        triOfShape[gp->shape.get()] = (int)f->materialId.size();
        f->materialId.push_back(mid);
        f->lightId.push_back(-1);
        return true;
    };
    std::vector<const TransformedPrimitive *> transformed;
    f->vertices.reserve(prims.size() * 9);
    for (size_t i = 0; i < prims.size(); ++i) {
        if (auto tp = dynamic_cast<const TransformedPrimitive *>(prims[i].get())) {
            transformed.push_back(tp);
            continue;
        }
        auto gp = dynamic_cast<const GeometricPrimitive *>(prims[i].get());
        if (!gp) return *why = "a primitive other than GeometricPrimitive / TransformedPrimitive", false;
        if (!volumetric && (gp->mediumInterface.inside || gp->mediumInterface.outside)) return *why = "participating media", false;
        auto sph = dynamic_cast<const Sphere *>(gp->shape.get());
        const bool boundary = volumetric && sph && gp->mediumInterface.IsMediumTransition() && !gp->material;
        if (!boundary && !noTransition(gp)) return false;
        if (sph) {
            b200pt_sphere bs;
            memset(&bs, 0, sizeof(bs));
            memcpy(bs.object_to_world, sph->ObjectToWorld->m.m, sizeof(float) * 16);
            memcpy(bs.world_to_object, sph->WorldToObject->m.m, sizeof(float) * 16);
            bs.radius = sph->radius;
            bs.z_min = sph->zMin;  // the Sphere's own members (sphere.h:66-68); phi_max != 0 marks them valid
            bs.z_max = sph->zMax;
            bs.theta_min = sph->thetaMin;
            bs.theta_max = sph->thetaMax;
            bs.phi_max = sph->phiMax;
            if (!(sph->phiMax > 0)) return *why = "a sphere with phimax 0", false;
            if (boundary) {
                // `Material ""` under `MediumInterface "inside" "outside"`: no BSDF, the ray changes medium there
                if (gp->areaLight) return *why = "a medium boundary that is also an area light", false;
                if (!gp->mediumInterface.inside) return *why = "a medium boundary with vacuum inside", false;
                if (kSampledHost) return *why = "media bounded by surfaces in a SampledSpectrum build", false;
                bs.material_id = 0;  // never looked at; the scene gets a material 0 below if it has none
                f->sphereMedium.resize(f->spheres.size(), -1);
                f->sphereMedium.push_back((int32_t)f->boundedMedia.size());
                f->boundedMedia.push_back(gp->mediumInterface.inside);
                f->boundaryOutside.push_back(gp->mediumInterface.outside);
            } else if (!materialOf(gp->material.get(), &bs.material_id))
                return false;
            bs.light_id = -1;
            bs.reverse_orientation = sph->reverseOrientation ? 1 : 0;
            bs.transform_swaps_handedness = sph->transformSwapsHandedness ? 1 : 0;
            sphereOfShape[gp->shape.get()] = (int)f->spheres.size();
            f->spheres.push_back(bs);
            continue;
        }
        if (!appendTriangle(gp)) return false;
    }
    f->nTopLevel = (int64_t)f->materialId.size();
    if (!f->boundedMedia.empty()) {
        f->sphereMedium.resize(f->spheres.size(), -1);
        if (!transformed.empty()) return *why = "media bounded by surfaces together with object instances", false;
        if (f->materials.empty()) {  // only boundaries: material id 0 must exist for the descriptor to validate
            b200pt_material bm;
            memset(&bm, 0, sizeof(bm));
            bm.type = B200PT_MAT_MATTE;
            f->materials.push_back(bm);
        }
    }
    // object instances (TransformedPrimitive, primitive.cpp:70-98): the triangles of every distinct object are appended
    // behind the top-level ones, in the object's own space
    std::unordered_map<const Primitive *, std::pair<int64_t, int64_t>> objectRange;
    std::unordered_map<const Primitive *, int> instanceOfPrim;
    for (const TransformedPrimitive *tp : transformed) {
        if (tp->PrimitiveToWorld.actuallyAnimated) return *why = "animated object instances", false;
        const Primitive *inner = tp->primitive.get();
        auto it = objectRange.find(inner);
        if (it == objectRange.end()) {
            const int64_t first = (int64_t)f->materialId.size();
            if (auto ob = dynamic_cast<const BVHAccel *>(inner)) {
                for (const auto &op : ob->primitives) {
                    auto ogp = dynamic_cast<const GeometricPrimitive *>(op.get());
                    if (!ogp) return *why = "nested instances", false;
                    if (ogp->areaLight) return *why = "area lights inside object instances", false;
                    if (!dynamic_cast<const Triangle *>(ogp->shape.get())) return *why = "non-triangle shapes inside object instances", false;
                    if (!appendTriangle(ogp)) return false;
                }
            } else if (auto ogp = dynamic_cast<const GeometricPrimitive *>(inner)) {
                if (!dynamic_cast<const Triangle *>(ogp->shape.get())) return *why = "non-triangle shapes inside object instances", false;
                if (!appendTriangle(ogp)) return false;
            } else {
                return *why = "object instances over an aggregate other than BVHAccel", false;
            }
            it = objectRange.emplace(inner, std::make_pair(first, (int64_t)f->materialId.size() - first)).first;
        }
        b200pt_instance bi;
        memset(&bi, 0, sizeof(bi));
        bi.first_triangle = it->second.first;
        bi.n_triangles = it->second.second;
        const Transform *t2w = tp->PrimitiveToWorld.startTransform;
        memcpy(bi.instance_to_world, t2w->m.m, sizeof(float) * 16);
        memcpy(bi.world_to_instance, t2w->mInv.m, sizeof(float) * 16);
        bi.is_identity = t2w->IsIdentity() ? 1 : 0;
        instanceOfPrim[tp] = (int)f->instances.size();
        f->instances.push_back(bi);
    }
    // the BVHAccel leaf of every sphere: its bounds gate Sphere::Intersect(P) in the reference (bvh.cpp:676,713)
    if ((!f->spheres.empty() || !f->instances.empty()) && bvh->nodes) {
        std::vector<int> stack(1, 0);
        while (!stack.empty()) {
            const int ni = stack.back();
            stack.pop_back();
            const LinearBVHNode &node = bvh->nodes[ni];
            if (node.nPrimitives > 0) {
                for (int i = 0; i < node.nPrimitives; ++i) {
                    auto ii = instanceOfPrim.find(prims[node.primitivesOffset + i].get());
                    if (ii != instanceOfPrim.end()) {
                        float *lb = f->instances[ii->second].leaf_bounds;
                        for (int a = 0; a < 3; ++a) {
                            lb[a] = node.bounds.pMin[a];
                            lb[3 + a] = node.bounds.pMax[a];
                        }
                        continue;
                    }
                    auto gp = dynamic_cast<const GeometricPrimitive *>(prims[node.primitivesOffset + i].get());
                    auto it = gp ? sphereOfShape.find(gp->shape.get()) : sphereOfShape.end();
                    if (it == sphereOfShape.end()) continue;
                    float *lb = f->spheres[it->second].leaf_bounds;
                    for (int a = 0; a < 3; ++a) {
                        lb[a] = node.bounds.pMin[a];
                        lb[3 + a] = node.bounds.pMax[a];
                    }
                }
            } else {
                stack.push_back(ni + 1);
                stack.push_back(node.secondChildOffset);
            }
        }
    }
    // Spectrum(RGBSpectrum, Illuminant) is a per-lookup FromRGB on SampledSpectrum hosts, which the device does not restate
    if (!scene.infiniteLights.empty() && kSampledHost) return *why = "infinite area lights in a SampledSpectrum build", false;
    if (!scene.infiniteLights.empty() && volumetric) return *why = "infinite area lights under the volumetric integrator", false;
    for (size_t l = 0; l < scene.lights.size(); ++l) {
        b200pt_area_light bl;
        memset(&bl, 0, sizeof(bl));
        bl.triangle = bl.sphere = -1;
        // delta lights (point.cpp:43-56, spot.cpp:42-76, distant.cpp:43-66): the lights' own members
        if (auto pl = dynamic_cast<const PointLight *>(scene.lights[l].get())) {
            bl.kind = B200PT_LIGHT_POINT;
            ToRGB(pl->I, bl.lemit, &f->lightSpectra);
            bl.position[0] = pl->pLight.x, bl.position[1] = pl->pLight.y, bl.position[2] = pl->pLight.z;
            f->lights.push_back(bl);
            continue;
        }
        if (auto sl = dynamic_cast<const SpotLight *>(scene.lights[l].get())) {
            bl.kind = B200PT_LIGHT_SPOT;
            ToRGB(sl->I, bl.lemit, &f->lightSpectra);
            bl.position[0] = sl->pLight.x, bl.position[1] = sl->pLight.y, bl.position[2] = sl->pLight.z;
            bl.cos_total_width = sl->cosTotalWidth;
            bl.cos_falloff_start = sl->cosFalloffStart;
            memcpy(bl.world_to_light, sl->WorldToLight.m.m, sizeof(float) * 16);
            f->lights.push_back(bl);
            continue;
        }
        if (auto tl = dynamic_cast<const DistantLight *>(scene.lights[l].get())) {
            bl.kind = B200PT_LIGHT_DISTANT;
            ToRGB(tl->L, bl.lemit, &f->lightSpectra);
            bl.position[0] = tl->wLight.x, bl.position[1] = tl->wLight.y, bl.position[2] = tl->wLight.z;
            bl.world_radius = tl->worldRadius;  // set by DistantLight::Preprocess in the Scene constructor
            f->lights.push_back(bl);
            continue;
        }
        if (auto il = dynamic_cast<const InfiniteAreaLight *>(scene.lights[l].get())) {
            // infinite.cpp:43-84: level 0 of Lmap (Le and Sample_Li look it up with width 0), the Distribution2D as built
            bl.kind = B200PT_LIGHT_INFINITE;
            memcpy(bl.world_to_light, il->WorldToLight.m.m, sizeof(float) * 16);
            bl.world_radius = il->worldRadius;  // set by InfiniteAreaLight::Preprocess in the Scene constructor
            Flattened::Infinite in;
            in.light = (int)l;
            const auto &lv0 = *il->Lmap->pyramid[0];
            in.width = lv0.uSize();
            in.height = lv0.vSize();
            for (int t = 0; t < in.height; ++t)
                for (int s = 0; s < in.width; ++s)
                    for (int c = 0; c < 3; ++c) in.texels.push_back(lv0(s, t)[c]);
            const Distribution2D &d2 = *il->distribution;
            in.nv = (int)d2.pConditionalV.size();
            in.nu = d2.pConditionalV[0]->Count();
            for (const auto &row : d2.pConditionalV) {
                in.condFunc.insert(in.condFunc.end(), row->func.begin(), row->func.end());
                in.condCdf.insert(in.condCdf.end(), row->cdf.begin(), row->cdf.end());
                in.condFuncInt.push_back(row->funcInt);
            }
            in.margFunc = d2.pMarginal->func;
            in.margCdf = d2.pMarginal->cdf;
            in.margFuncInt = d2.pMarginal->funcInt;
            memcpy(in.lightToWorld, il->LightToWorld.m.m, sizeof(float) * 16);
            const RGBSpectrum pw = il->Lmap->Lookup(Point2f(.5f, .5f), .5f);
            for (int c = 0; c < 3; ++c) in.powerRGB[c] = pw[c];
            f->infinite.push_back(std::move(in));
            f->lights.push_back(bl);
            continue;
        }
        auto dl = dynamic_cast<const DiffuseAreaLight *>(scene.lights[l].get());
        if (!dl) return *why = "a light other than diffuse area / point / spot / distant / infinite lights", false;
        ToRGB(dl->Lemit, bl.lemit, &f->lightSpectra);
        bl.two_sided = dl->twoSided ? 1 : 0;
        auto is = sphereOfShape.find(dl->shape.get());
        if (is != sphereOfShape.end()) {
            bl.triangle = -1;
            bl.sphere = is->second;
            f->spheres[is->second].light_id = (int)l;
            f->lights.push_back(bl);
            continue;
        }
        auto it = triOfShape.find(dl->shape.get());
        if (it == triOfShape.end()) return *why = "an area light on a shape that is not in the scene", false;
        bl.triangle = it->second;
        bl.sphere = -1;
        f->lightId[it->second] = (int)l;
        f->lights.push_back(bl);
    }
    return true;
}

}  // namespace

// Base = PathIntegrator (integrators/path.h:48-66) or VolPathIntegrator (integrators/volpath.h:49-66): the same members
// (maxDepth, rrThreshold, lightSampleStrategy), the same constructor signature, Render() replaced.
template <class Base>
class GpuIntegrator : public Base {
    static constexpr bool kVolumetric = std::is_same<Base, VolPathIntegrator>::value;

  public:
    GpuIntegrator(int maxDepth, std::shared_ptr<const Camera> camera, std::shared_ptr<Sampler> sampler,
                  const Bounds2i &pixelBounds, Float rrThreshold, const std::string &lightSampleStrategy)
        : Base(maxDepth, camera, sampler, pixelBounds, rrThreshold, lightSampleStrategy),
          cam(camera),
          smp(sampler),
          bounds(pixelBounds) {}

    void Render(const Scene &scene) override {
#define B200_CHECK(call)                                                            \
    do {                                                                            \
        if ((call) != B200PT_OK) {                                                  \
            Error("gpupath: %s failed: %s", #call, b200pt_last_error());            \
            return;                                                                 \
        }                                                                           \
    } while (0)
        std::string why;
        auto pcam = dynamic_cast<const PerspectiveCamera *>(cam.get());
        if (!pcam) return Error("gpupath: only the perspective camera is supported");
        if (pcam->CameraToWorld.actuallyAnimated) return Error("gpupath: animated cameras are not supported");
        auto sobol = dynamic_cast<const SobolSampler *>(smp.get());
        auto halton = dynamic_cast<const HaltonSampler *>(smp.get());
        if (!sobol && !halton) return Error("gpupath: only Sampler \"sobol\" and \"halton\" are supported");
        if (halton && halton->sampleAtPixelCenter)
            return Error("gpupath: Sampler \"halton\" with samplepixelcenter is not supported");
        Film *film = cam->film;
        if (film->filter->radius.x > 8 || film->filter->radius.y > 8)
            return Error("gpupath: pixel filters wider than 8 pixels are not supported");
        int strategy;
        const std::string &lightSampleStrategy = this->lightSampleStrategy;
        const int maxDepth = this->maxDepth;
        const Float rrThreshold = this->rrThreshold;
        if (lightSampleStrategy == "uniform" || scene.lights.size() == 1)
            strategy = B200PT_LIGHTS_UNIFORM;
        else if (lightSampleStrategy == "power")
            strategy = B200PT_LIGHTS_POWER;
        else  // "spatial" and, like the reference (lightdistrib.cpp:59-65), any unknown name
            strategy = B200PT_LIGHTS_SPATIAL;
        Flattened flat;
        if (!FlattenScene(scene, &flat, &why, kVolumetric)) return Error("gpupath: the scene uses %s", why.c_str());

        b200pt_scene_desc sd;
        memset(&sd, 0, sizeof(sd));
        sd.n_triangles = (int64_t)flat.materialId.size();
        sd.vertices = flat.vertices.data();
        sd.material_id = flat.materialId.data();
        sd.light_id = flat.lightId.data();
        sd.flip_normal = flat.flip.data();
        sd.n_materials = (int)flat.materials.size();
        sd.materials = flat.materials.data();
        sd.n_lights = (int)flat.lights.size();
        sd.lights = flat.lights.data();
        sd.normals = flat.anyNormals ? flat.normals.data() : nullptr;
        sd.uvs = flat.anyUVs ? flat.uvs.data() : nullptr;
        sd.vertex_flags = flat.vertexFlags.data();
        sd.n_spheres = (int)flat.spheres.size();
        sd.spheres = flat.spheres.data();
        sd.n_instances = (int)flat.instances.size();
        sd.instances = flat.instances.data();
        sd.n_toplevel_triangles = flat.nTopLevel;
        std::vector<float> cie;
        if (kSampledHost) {  // spectrum.cpp:80-100: the CIE matching curves averaged over the bins at SampledSpectrum::Init
            for (const SampledSpectrum *c : {&SampledSpectrum::X, &SampledSpectrum::Y, &SampledSpectrum::Z})
                for (int i = 0; i < SampledSpectrum::nSamples; ++i) cie.push_back((*c)[i]);
            sd.n_spectrum_samples = Spectrum::nSamples;
            sd.material_spectra = flat.materialSpectra.data();
            sd.light_spectra = flat.lightSpectra.data();
            sd.cie_xyz = cie.data();
        }

        b200pt_camera_desc cd;
        memcpy(cd.raster_to_camera, pcam->RasterToCamera.m.m, sizeof(float) * 16);
        memcpy(cd.camera_to_world, pcam->CameraToWorld.startTransform->m.m, sizeof(float) * 16);
        cd.lens_radius = pcam->lensRadius;
        cd.focal_distance = pcam->focalDistance;
        cd.shutter_open = pcam->shutterOpen;
        cd.shutter_close = pcam->shutterClose;

        b200pt_film_desc fd;
        fd.full_resolution[0] = film->fullResolution.x;
        fd.full_resolution[1] = film->fullResolution.y;
        const Bounds2i cb = film->croppedPixelBounds;
        fd.cropped_bounds[0] = cb.pMin.x;
        fd.cropped_bounds[1] = cb.pMin.y;
        fd.cropped_bounds[2] = cb.pMax.x;
        fd.cropped_bounds[3] = cb.pMax.y;
        fd.filter_radius[0] = film->filter->radius.x;
        fd.filter_radius[1] = film->filter->radius.y;
        fd.scale = film->scale;
        fd.max_sample_luminance = film->maxSampleLuminance;
        // any Filter: Film already tabulated it (film.cpp:68-77); the default box filter keeps the specialised path
        const bool defaultBox = dynamic_cast<const BoxFilter *>(film->filter.get()) && film->filter->radius.x == 0.5f &&
                                film->filter->radius.y == 0.5f;
        fd.filter_table = defaultBox ? nullptr : film->filterTable;

        b200pt_sampler_desc smpd;
        memset(&smpd, 0, sizeof(smpd));
        smpd.samples_per_pixel = (int32_t)smp->samplesPerPixel;
        // both samplers are constructed from Film::GetSampleBounds() (api.cpp:820-831); Halton keeps
        // only what it derives from them
        const Bounds2i sb = sobol ? sobol->sampleBounds : film->GetSampleBounds();
        smpd.sample_bounds[0] = sb.pMin.x;
        smpd.sample_bounds[1] = sb.pMin.y;
        smpd.sample_bounds[2] = sb.pMax.x;
        smpd.sample_bounds[3] = sb.pMax.y;
        if (sobol) {
            smpd.type = B200PT_SAMPLER_SOBOL;
            smpd.n_dimensions = NumSobolDimensions;
            smpd.matrices32 = SobolMatrices32;
            const int row = std::max(sobol->log2Resolution - 1, 0);
            smpd.vdc = VdCSobolMatrices[row];
            smpd.vdc_inv = VdCSobolMatricesInv[row];
        } else {
            smpd.type = B200PT_SAMPLER_HALTON;
            smpd.n_dimensions = PrimeTableSize;
            smpd.halton_permutations = HaltonSampler::radicalInversePermutations.data();
        }

        b200pt_integrator_desc id;
        memset(&id, 0, sizeof(id));
        std::vector<float> mediumSpectra;
        if (kVolumetric) {
            // VolPathIntegrator: the camera ray's medium (camera.h:76) is every ray's medium when no surface is a medium
            // transition (checked while flattening); only HomogeneousMedium is supported
            id.volumetric = 1;
            if (const Medium *m = cam->medium) {
                auto hm = dynamic_cast<const HomogeneousMedium *>(m);
                if (!hm) return Error("gpupath: only homogeneous media are supported");
                id.medium.present = 1;
                mediumSpectra.assign(2 * (size_t)B200PT_SPECTRUM_SAMPLES, 0.f);
                ToRGB(hm->sigma_a, id.medium.sigma_a, mediumSpectra.data());
                ToRGB(hm->sigma_s, id.medium.sigma_s, mediumSpectra.data() + B200PT_SPECTRUM_SAMPLES);
                if (kSampledHost) id.medium.spectra = mediumSpectra.data();  // the 60 bins of sigma_a, sigma_s
                id.medium.g = hm->g;
            }
        }
        // media bounded by null-material spheres: the medium inside each, all of them inside the camera's medium (or vacuum)
        std::vector<b200pt_medium> boundedMedia(flat.boundedMedia.size());
        for (size_t k = 0; k < flat.boundedMedia.size(); ++k) {
            auto hm = dynamic_cast<const HomogeneousMedium *>(flat.boundedMedia[k]);
            if (!hm) return Error("gpupath: only homogeneous media are supported");
            if (flat.boundaryOutside[k] != cam->medium)
                return Error("gpupath: a medium boundary whose outside is not the camera's medium");
            memset(&boundedMedia[k], 0, sizeof(b200pt_medium));
            boundedMedia[k].present = 1;
            ToRGB(hm->sigma_a, boundedMedia[k].sigma_a);
            ToRGB(hm->sigma_s, boundedMedia[k].sigma_s);
            boundedMedia[k].g = hm->g;
        }
        if (!boundedMedia.empty()) {
            id.n_bounded_media = (int32_t)boundedMedia.size();
            id.bounded_media = boundedMedia.data();
            id.sphere_medium = flat.sphereMedium.data();
        }
        id.max_depth = maxDepth;
        id.rr_threshold = rrThreshold;
        id.light_strategy = strategy;
        id.pixel_bounds[0] = bounds.pMin.x;
        id.pixel_bounds[1] = bounds.pMin.y;
        id.pixel_bounds[2] = bounds.pMax.x;
        id.pixel_bounds[3] = bounds.pMax.y;

        // B200PT_DUMP_SCENE=<file>: write the descriptors handed to the C ABI (debugging aid: the Python harness
        // can replay exactly what this host passes, see tests/replay_dump.py)
        if (const char *dp = getenv("B200PT_DUMP_SCENE")) {
            if (FILE *df = fopen(dp, "wb")) {
                const int64_t hdr[8] = {0x3154504d55443042ll, sd.n_triangles, sd.n_materials, sd.n_lights, sd.n_spheres,
                                        sd.normals != nullptr, sd.uvs != nullptr, (int64_t)smpd.type};
                fwrite(hdr, 8, 8, df);
                fwrite(sd.vertices, 4, (size_t)sd.n_triangles * 9, df);
                fwrite(sd.material_id, 4, (size_t)sd.n_triangles, df);
                fwrite(sd.light_id, 4, (size_t)sd.n_triangles, df);
                fwrite(sd.flip_normal, 1, (size_t)sd.n_triangles, df);
                fwrite(sd.vertex_flags, 1, (size_t)sd.n_triangles, df);
                if (sd.normals) fwrite(sd.normals, 4, (size_t)sd.n_triangles * 9, df);
                if (sd.uvs) fwrite(sd.uvs, 4, (size_t)sd.n_triangles * 6, df);
                fwrite(sd.materials, sizeof(b200pt_material), (size_t)sd.n_materials, df);
                fwrite(sd.lights, sizeof(b200pt_area_light), (size_t)sd.n_lights, df);
                fwrite(sd.spheres, sizeof(b200pt_sphere), (size_t)sd.n_spheres, df);
                fwrite(&cd, sizeof(cd), 1, df);
                fwrite(&fd, sizeof(fd), 1, df);
                fwrite(&id, sizeof(id), 1, df);
                const int32_t sm[6] = {smpd.samples_per_pixel, smpd.sample_bounds[0], smpd.sample_bounds[1],
                                       smpd.sample_bounds[2], smpd.sample_bounds[3], smpd.n_dimensions};
                fwrite(sm, 4, 6, df);
                // trailer of a SampledSpectrum host: bin count, then the three tables
                const int32_t ns = sd.n_spectrum_samples;
                fwrite(&ns, 4, 1, df);
                if (ns) {
                    fwrite(sd.material_spectra, 4, (size_t)sd.n_materials * B200PT_MATERIAL_SPECTRA * ns, df);
                    fwrite(sd.light_spectra, 4, (size_t)sd.n_lights * ns, df);
                    fwrite(sd.cie_xyz, 4, (size_t)3 * ns, df);
                }
                // infinite lights (appended after the layout above): light index, map and distribution sizes, the tables
                for (const auto &in : flat.infinite) {
                    const int32_t sz[5] = {in.light, in.width, in.height, in.nu, in.nv};
                    fwrite(sz, 4, 5, df);
                    fwrite(in.texels.data(), 4, in.texels.size(), df);
                    fwrite(in.lightToWorld, 4, 16, df);
                    fwrite(in.condFunc.data(), 4, in.condFunc.size(), df);
                    fwrite(in.condCdf.data(), 4, in.condCdf.size(), df);
                    fwrite(in.condFuncInt.data(), 4, in.condFuncInt.size(), df);
                    fwrite(in.margFunc.data(), 4, in.margFunc.size(), df);
                    fwrite(in.margCdf.data(), 4, in.margCdf.size(), df);
                    fwrite(&in.margFuncInt, 4, 1, df);
                    fwrite(in.powerRGB, 4, 3, df);
                }
                // image textures (appended after the infinite lights, behind a negative marker): the MIPMaps, then the bindings
                if (!flat.binds.empty()) {
                    const int32_t th[3] = {-2, (int32_t)flat.mipmaps.size(), (int32_t)flat.binds.size()};
                    fwrite(th, 4, 3, df);
                    for (const auto &m : flat.mipmaps) {
                        const int32_t mh[4] = {(int32_t)m.levels.size(), m.channels, m.wrap, m.trilinear};
                        fwrite(mh, 4, 4, df);
                        fwrite(&m.maxAniso, 4, 1, df);
                        fwrite(m.weightLut, 4, 128, df);
                        for (size_t l = 0; l < m.levels.size(); ++l) {
                            const int32_t wh[2] = {m.w[l], m.h[l]};
                            fwrite(wh, 4, 2, df);
                            fwrite(m.levels[l].data(), 4, m.levels[l].size(), df);
                        }
                    }
                    for (const auto &b : flat.binds) {
                        const int32_t bi[3] = {b.material, b.slot, b.mip};
                        const float bf[4] = {b.su, b.sv, b.du, b.dv};
                        fwrite(bi, 4, 3, df);
                        fwrite(bf, 4, 4, df);
                        fwrite(&b.remap, 4, 1, df);
                    }
                }
                // alpha masks (appended after the texture tables, behind their own marker): the masks, then per triangle
                // the alpha and the shadowalpha mask ids
                if (!flat.alphaMasks.empty()) {
                    const int32_t ah[2] = {-3, (int32_t)flat.alphaMasks.size()};
                    fwrite(ah, 4, 2, df);
                    for (const auto &a : flat.alphaMasks) {
                        const int32_t mh[3] = {a.w, a.h, a.wrap};
                        const float mf[4] = {a.su, a.sv, a.du, a.dv};
                        fwrite(mh, 4, 3, df);
                        fwrite(mf, 4, 4, df);
                        fwrite(a.texels.data(), 4, a.texels.size(), df);
                    }
                    fwrite(flat.alphaId.data(), 4, flat.alphaId.size(), df);
                    fwrite(flat.shadowAlphaId.data(), 4, flat.shadowAlphaId.size(), df);
                }
                fclose(df);
            }
        }
        const int device = getenv("B200PT_DEVICE") ? atoi(getenv("B200PT_DEVICE")) : 0;
        b200pt_ctx *ctx = nullptr;
        b200pt_scene *gscene = nullptr;
        b200pt_render *render = nullptr;
        // whatever way this function is left (B200_CHECK returns on the first failing call), the device objects go with it
        struct Handles {
            b200pt_ctx *&c;
            b200pt_scene *&s;
            b200pt_render *&r;
            ~Handles() {
                if (r) b200pt_render_destroy(r);
                if (s) b200pt_scene_destroy(s);
                if (c) b200pt_ctx_destroy(c);
            }
        } handles{ctx, gscene, render};
        auto now = []() { return std::chrono::steady_clock::now(); };
        auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
            return std::chrono::duration<double, std::milli>(b - a).count();
        };
        const auto t0 = now();
        B200_CHECK(b200pt_ctx_create(device, &ctx));
        const auto t1 = now();
        B200_CHECK(b200pt_scene_create(ctx, &sd, &gscene));
        for (const auto &in : flat.infinite) {
            b200pt_infinite_light il;
            memset(&il, 0, sizeof(il));
            il.width = in.width;
            il.height = in.height;
            il.texels = in.texels.data();
            memcpy(il.light_to_world, in.lightToWorld, sizeof(il.light_to_world));
            il.nu = in.nu;
            il.nv = in.nv;
            il.cond_func = in.condFunc.data();
            il.cond_cdf = in.condCdf.data();
            il.cond_func_int = in.condFuncInt.data();
            il.marg_func = in.margFunc.data();
            il.marg_cdf = in.margCdf.data();
            il.marg_func_int = in.margFuncInt;
            memcpy(il.power_rgb, in.powerRGB, sizeof(il.power_rgb));
            B200_CHECK(b200pt_scene_set_infinite_light(gscene, in.light, &il));
        }
        std::vector<int32_t> mipIds;
        for (const auto &m : flat.mipmaps) {
            b200pt_mipmap bm;
            memset(&bm, 0, sizeof(bm));
            if (m.levels.size() > B200PT_MIPMAP_MAX_LEVELS) return Error("gpupath: image textures larger than %d texels on a side are not supported", 1 << (B200PT_MIPMAP_MAX_LEVELS - 1));
            bm.n_levels = (int32_t)m.levels.size();
            bm.channels = m.channels;
            for (size_t l = 0; l < m.levels.size(); ++l) {
                bm.width[l] = m.w[l];
                bm.height[l] = m.h[l];
                bm.texels[l] = m.levels[l].data();
            }
            bm.wrap = m.wrap;
            bm.trilinear = m.trilinear;
            bm.max_anisotropy = m.maxAniso;
            memcpy(bm.weight_lut, m.weightLut, sizeof(bm.weight_lut));
            int32_t mid = -1;
            B200_CHECK(b200pt_scene_add_mipmap(gscene, &bm, &mid));
            mipIds.push_back(mid);
        }
        for (const auto &b : flat.binds)
            B200_CHECK(b200pt_scene_bind_texture(gscene, b.material, b.slot, mipIds[b.mip], b.su, b.sv, b.du, b.dv, b.remap));
        if (!flat.alphaMasks.empty()) {
            for (const auto &a : flat.alphaMasks) {
                b200pt_alpha_mask am;
                memset(&am, 0, sizeof(am));
                am.width = a.w;
                am.height = a.h;
                am.texels = a.w ? a.texels.data() : nullptr;
                am.wrap = a.wrap;
                am.su = a.su;
                am.sv = a.sv;
                am.du = a.du;
                am.dv = a.dv;
                int32_t aid = -1;
                B200_CHECK(b200pt_scene_add_alpha_mask(gscene, &am, &aid));  // ids follow the order of the calls
            }
            B200_CHECK(b200pt_scene_set_alpha_masks(gscene, flat.alphaId.data(), flat.shadowAlphaId.data()));
        }
        B200_CHECK(b200pt_render_create(gscene, &cd, &fd, &smpd, &id, &render));
        B200_CHECK(b200pt_ctx_synchronize(ctx));
        const auto t2 = now();
        int32_t nx = 0, ny = 0;
        B200_CHECK(b200pt_render_tile_counts(render, &nx, &ny));
        // image-space sharding across processes (one per GPU): rank r renders tiles r, r+N, ...
        const int rank = getenv("B200PT_RANK") ? atoi(getenv("B200PT_RANK")) : 0;
        const int world = getenv("B200PT_WORLD_SIZE") ? std::max(1, atoi(getenv("B200PT_WORLD_SIZE"))) : 1;
        std::vector<int32_t> tiles;
        for (int32_t t = rank; t < nx * ny; t += world) tiles.push_back(t);
        // B200PT_REPEAT=n renders n times (film cleared in between) so that a launcher can time a warm render
        const int repeat = getenv("B200PT_REPEAT") ? std::max(1, atoi(getenv("B200PT_REPEAT"))) : 1;
        double renderMs = 0;
        {
            ProgressReporter reporter(1, "Rendering (GPU)");
            for (int it = 0; it < repeat; ++it) {
                if (it) B200_CHECK(b200pt_film_clear(render));
                B200_CHECK(b200pt_reset_stats(render));
                B200_CHECK(b200pt_ctx_synchronize(ctx));
                const auto ta = now();
                B200_CHECK(b200pt_render_tiles(render, tiles.data(), (int64_t)tiles.size()));
                B200_CHECK(b200pt_ctx_synchronize(ctx));
                renderMs = ms(ta, now());
            }
            reporter.Update();
            reporter.Done();
        }
        // raw film sums -> Film::pixels (film.h:83-89), then the reference's own WriteImage
        const int w = cb.pMax.x - cb.pMin.x, h = cb.pMax.y - cb.pMin.y;
        std::vector<float> raw((size_t)w * h * 4);
        // Several processes (B200PT_RANK / B200PT_WORLD_SIZE, one per GPU) rendered disjoint tile sets of this film:
        // their raw sums meet on rank 0, the only rank that writes the image.  With B200PT_NCCL_ID_FILE (a fresh path
        // every rank can reach, chosen by the launcher) it is one ncclReduce over NVLink behind the C ABI
        // (b200pt_film_reduce); otherwise -- or if NCCL cannot start, e.g. two ranks on one GPU -- the ranks hand their
        // raw films to rank 0 through files next to the image.  The reference's equivalent is `imgtool assemble`
        // (tools/imgtool.cpp:190-285) after independent crop-window runs.
        bool merged = world == 1;
        if (!merged && getenv("B200PT_NCCL_ID_FILE")) {
            b200pt_comm *comm = nullptr;
            if (b200pt_comm_create(ctx, rank, world, getenv("B200PT_NCCL_ID_FILE"), &comm) == B200PT_OK) {
                B200_CHECK(b200pt_film_reduce(render, comm, 0));
                B200_CHECK(b200pt_ctx_synchronize(ctx));
                b200pt_comm_destroy(comm);
                merged = true;
            } else {
                Warning("gpupath: NCCL film reduce unavailable (%s); merging through files", b200pt_last_error());
            }
        }
        B200_CHECK(b200pt_film_read_raw(render, raw.data()));
        if (!merged) {
            auto part = [&](int k) { return film->filename + ".rank" + std::to_string(k) + ".raw"; };
            if (rank != 0) {
                const std::string tmp = part(rank) + ".tmp";
                FILE *f = fopen(tmp.c_str(), "wb");
                if (!f || fwrite(raw.data(), sizeof(float), raw.size(), f) != raw.size()) {
                    Error("gpupath: cannot write %s", tmp.c_str());
                    if (f) fclose(f);
                } else {
                    fclose(f);
                    rename(tmp.c_str(), part(rank).c_str());
                }
            } else {
                std::vector<float> other(raw.size());
                for (int k = 1; k < world; ++k) {  // rank order: the sum is reproducible
                    bool got = false;
                    for (int tries = 0; tries < 72000 && !got; ++tries) {  // up to an hour for the slowest rank
                        if (FILE *f = fopen(part(k).c_str(), "rb")) {
                            got = fread(other.data(), sizeof(float), other.size(), f) == other.size();
                            fclose(f);
                        }
                        if (!got) std::this_thread::sleep_for(std::chrono::milliseconds(50));
                    }
                    if (!got) {
                        Error("gpupath: rank %d's film %s never arrived; the image holds the other ranks' tiles only", k, part(k).c_str());
                        continue;
                    }
                    for (size_t i = 0; i < raw.size(); ++i) raw[i] += other[i];
                    remove(part(k).c_str());
                }
            }
        }
        for (size_t i = 0; i < (size_t)w * h; ++i) {
            Film::Pixel &p = film->pixels[i];
            p.xyz[0] = raw[4 * i];
            p.xyz[1] = raw[4 * i + 1];
            p.xyz[2] = raw[4 * i + 2];
            p.filterWeightSum = raw[4 * i + 3];
        }
        b200pt_stats st;
        if (b200pt_get_stats(render, &st) == B200PT_OK) {
            nGpuCameraRays += st.camera_rays;
            nGpuRegular += st.regular_rays;
            nGpuShadow += st.shadow_rays;
            // B200PT_REPORT=<file>: one JSON line with the timings of this render (bench.py --workload cfg1)
            if (const char *rp = getenv("B200PT_REPORT")) {
                if (FILE *rf = fopen(rp, "w")) {
                    fprintf(rf,
                            "{\"triangles\": %lld, \"spheres\": %d, \"lights\": %d, \"camera_rays\": %llu, "
                            "\"regular_rays\": %llu, \"shadow_rays\": %llu, \"ctx_ms\": %.3f, \"scene_build_upload_ms\": %.3f, "
                            "\"render_ms\": %.3f, \"launches\": %llu}\n",
                            (long long)sd.n_triangles, sd.n_spheres, sd.n_lights, (unsigned long long)st.camera_rays,
                            (unsigned long long)st.regular_rays, (unsigned long long)st.shadow_rays, ms(t0, t1), ms(t1, t2),
                            renderMs, (unsigned long long)st.launches);
                    fclose(rf);
                }
            }
        }
        b200pt_render_destroy(render);
        render = nullptr;
        b200pt_scene_destroy(gscene);
        gscene = nullptr;
        b200pt_ctx_destroy(ctx);
        ctx = nullptr;
        if (rank == 0) film->WriteImage();  // the other ranks' tiles are part of rank 0's image
#undef B200_CHECK
    }

  private:
    std::shared_ptr<const Camera> cam;
    std::shared_ptr<Sampler> smp;
    const Bounds2i bounds;
};

// integrators/path.cpp:190-213 -- same parameters, same defaults.
PathIntegrator *CreatePathIntegrator(const ParamSet &params, std::shared_ptr<Sampler> sampler,
                                     std::shared_ptr<const Camera> camera) {
    int maxDepth = params.FindOneInt("maxdepth", 5);
    int np;
    const int *pb = params.FindInt("pixelbounds", &np);
    Bounds2i pixelBounds = camera->film->GetSampleBounds();
    if (pb) {
        if (np != 4)
            Error("Expected four values for \"pixelbounds\" parameter. Got %d.", np);
        else {
            pixelBounds = Intersect(pixelBounds, Bounds2i{{pb[0], pb[2]}, {pb[1], pb[3]}});
            if (pixelBounds.Area() == 0) Error("Degenerate \"pixelbounds\" specified.");
        }
    }
    Float rrThreshold = params.FindOneFloat("rrthreshold", 1.);
    std::string lightStrategy = params.FindOneString("lightsamplestrategy", "spatial");
    return new GpuIntegrator<PathIntegrator>(maxDepth, camera, sampler, pixelBounds, rrThreshold, lightStrategy);
}

// integrators/volpath.cpp:190-214 -- same parameters, same defaults.  `Integrator "volpath"` renders on the GPU when the
// scene's media are at most one homogeneous medium around everything (the camera's medium, no medium transitions).
VolPathIntegrator *CreateVolPathIntegrator(const ParamSet &params, std::shared_ptr<Sampler> sampler,
                                           std::shared_ptr<const Camera> camera) {
    int maxDepth = params.FindOneInt("maxdepth", 5);
    int np;
    const int *pb = params.FindInt("pixelbounds", &np);
    Bounds2i pixelBounds = camera->film->GetSampleBounds();
    if (pb) {
        if (np != 4)
            Error("Expected four values for \"pixelbounds\" parameter. Got %d.", np);
        else {
            pixelBounds = Intersect(pixelBounds, Bounds2i{{pb[0], pb[2]}, {pb[1], pb[3]}});
            if (pixelBounds.Area() == 0) Error("Degenerate \"pixelbounds\" specified.");
        }
    }
    Float rrThreshold = params.FindOneFloat("rrthreshold", 1.);
    std::string lightStrategy = params.FindOneString("lightsamplestrategy", "spatial");
    return new GpuIntegrator<VolPathIntegrator>(maxDepth, camera, sampler, pixelBounds, rrThreshold, lightStrategy);
}

}  // namespace pbrt
