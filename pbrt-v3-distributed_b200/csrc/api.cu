// api.cu -- implementation of the C ABI (include/b200pt.h): contexts, scene
// upload (+ host BVH build), the wavefront batch driver and film read-back.
// Host code only orchestrates; all arithmetic of the path runs in kernels.cu.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <string>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "b200pt_internal.h"
#include "wbvh.h"
#include "wbvh_gpu.h"
#include "kernels.cuh"

using namespace b200pt;

#define CUDA_TRY(expr)                                                                                    \
    do {                                                                                                  \
        cudaError_t e_ = (expr);                                                                          \
        if (e_ != cudaSuccess)                                                                            \
            return b200pt_fail(e_ == cudaErrorMemoryAllocation ? B200PT_ERR_OOM : B200PT_ERR_CUDA,       \
                               "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

struct b200pt_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t stream_aux = nullptr;   // shadow / MIS rays of bounce b overlap the path rays of bounce b+1
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    int sm_count = 0;
    bool gpu_bvh_build = false;  // b200pt_ctx_set_option "gpu_bvh_build"
};

// Entry points of the SampledSpectrum translation unit (kernels.cu compiled with B200PT_NSPEC 60, see the Makefile).
// Its RenderDev is the struct of kernels.cuh again -- no member depends on the spectrum type -- so this file hands
// over its own RenderDev objects (render_dev_size() is checked once per render object).
namespace b200pt_s60 {
struct RenderDev;
void launch_raygen(const RenderDev *dev, uint32_t batch_first_tile, uint32_t n_batch_tiles, uint32_t n_slots, cudaStream_t s);
void launch_shade(const RenderDev *dev, int material, bool vertex_data, int bounce, uint32_t *work, int grid, cudaStream_t s);
void launch_resolve(const RenderDev *dev, int bounce, uint32_t *work, int grid, cudaStream_t s);
void launch_medium(const RenderDev *dev, int bounce, uint32_t *work, int grid, cudaStream_t s);
void launch_spatial_build(const RenderDev *dev, const RenderDev &host, cudaStream_t s);
void launch_film(const RenderDev *dev, uint32_t batch_first_tile, uint32_t n_batch_tiles, cudaStream_t s);
void launch_film_general(const RenderDev *dev, const RenderDev &host, uint32_t batch_first_tile, uint32_t n_batch_tiles,
                         cudaStream_t s);
void set_cie_xyz(const float *xyz, cudaStream_t s);
size_t render_dev_size();
}  // namespace b200pt_s60
static inline const b200pt_s60::RenderDev *s60(const RenderDev *p) { return reinterpret_cast<const b200pt_s60::RenderDev *>(p); }
static inline const b200pt_s60::RenderDev &s60(const RenderDev &p) { return reinterpret_cast<const b200pt_s60::RenderDev &>(p); }

struct b200pt_scene {
    b200pt_ctx *ctx = nullptr;
    U4 *d_nodes = nullptr;       // WbvhNode[n_nodes] (wbvh.h), the top-level tree first, then the objects' trees, then the tree over the instances
    uint32_t *d_tri_base = nullptr;  // per node: first triangle of its leaf children
    uint8_t *d_lut = nullptr;    // permute_slots table of the node test (wbvh_traverse.cuh)
    TravBounds trav_bounds, tlas_bounds;  // padded bounds of the top-level tree / of the tree over the instances
    F4 *d_tris = nullptr;
    b200pt_material *d_materials = nullptr;
    F4 *d_tri_n = nullptr, *d_tri_uv = nullptr;
    uint64_t n_nodes = 0, n_tris = 0;
    uint64_t n_top_nodes = 0;  // nodes of the top-level tree (the first ones of d_nodes)
    std::vector<b200pt_material> materials;
    std::vector<b200pt_area_light> lights;  // host copy, triangle = original index
    std::vector<uint32_t> prim_to_tri;
    std::vector<float> light_area;
    float bounds_lo[3] = {0, 0, 0}, bounds_hi[3] = {0, 0, 0};
    std::vector<DevSphere> spheres;  // Sphere shapes (tested outside the BVH)
    DevSphere *d_spheres = nullptr;
    std::vector<DevInstance> instances;  // object instances (tested by the same pass as the spheres)
    DevInstance *d_instances = nullptr;
    uint32_t tlas_node_off = 0, tlas_tri_off = 0;  // tree over the instances' leaf boxes inside the node / triangle arrays
    uint64_t n_prims = 0;            // triangles of the descriptor (sphere k is reported as primitive n_prims + k)
    uint32_t *d_work = nullptr;  // fetch counter for the ray-batch entry points
    void *h_nodes = nullptr, *h_tris = nullptr, *h_tri_base = nullptr;  // pinned host copies (b200pt_scene_upload)
    // SampledSpectrum hosts (b200pt_scene_desc::n_spectrum_samples == 60): host copies of the tables
    int nspec = 0;
    std::vector<float> material_spectra, light_spectra, cie_xyz;
    float *d_material_spectra = nullptr;
};

struct TimedLaunch {
    cudaEvent_t a, b;
    int category;  // 0 closest, 1 any, 2 other
};

struct b200pt_render {
    b200pt_scene *scene = nullptr;
    RenderDev host;           // host copy of the device parameter block
    RenderDev *d_dev = nullptr;
    std::vector<void *> allocs;
    b200pt_film_desc film;
    int spp = 0;
    uint32_t tiles_per_batch = 1;
    int32_t *d_tile_list = nullptr;
    size_t tile_list_capacity = 0;
    float *d_rgb = nullptr;  // b200pt_film_read_rgb staging (lazily allocated, freed with the render object)
    uint32_t *d_walk_counts = nullptr;  // bounded media: [16] queue counters / fetch counters of the boundary passes
    int grid_trace = 0, grid_shade = 0, grid_shade_s60 = 0;
    bool instrumented = false, profiling = false;
    int refill_lanes = 26, postpone_pct = 40, trace_ctas = 0, stage_nodes = 0;  // k_trace knobs (b200pt_render_set_option)
    bool overlap = true;  // run shadow/MIS rays of bounce b concurrently with the path rays of bounce b+1
    int sort_from_bounce = -1;  // coherence-sort the path / shadow queues from this bounce on (<0: never; measured: no gain on the soups)
    std::vector<TimedLaunch> timed;
    std::vector<cudaEvent_t> event_pool;
    double ms[3] = {0, 0, 0};
    uint64_t launches = 0, launches_cat[3] = {0, 0, 0};
};

// Host restatement of Spectrum::y() for the light-power distribution (Light::Power().y(), integrator.cpp:216-224):
// RGBSpectrum (spectrum.h:462-465) or SampledSpectrum (spectrum.h:393-398) with the host's Y curve.
static float host_spectrum_y(const b200pt_scene *sc, const std::vector<float> &c) {
    if (!sc->nspec) return 0.212671f * c[0] + 0.715160f * c[1] + 0.072169f * c[2];
    const float *Y = sc->cie_xyz.data() + sc->nspec;
    float yy = 0.f;
    for (int i = 0; i < sc->nspec; ++i) yy += Y[i] * c[i];
    return yy * float(700 - 400) / float(106.856895f * sc->nspec);  // (yy * range) / (integral * n), in this order
}
// Lemit / I / L of light i as the host holds it
static std::vector<float> host_light_spectrum(const b200pt_scene *sc, int i) {
    if (!sc->nspec) return std::vector<float>(sc->lights[i].lemit, sc->lights[i].lemit + 3);
    return std::vector<float>(sc->light_spectra.begin() + (size_t)i * sc->nspec, sc->light_spectra.begin() + (size_t)(i + 1) * sc->nspec);
}

// Bounds a ray is clipped to before it walks a tree (trav_init): the tree's own bounds padded by a few of its
// smallest cells, so that no triangle on the boundary is lost to the rounding of that clip.
static TravBounds make_trav_bounds(const float *lo, const float *hi) {
    TravBounds b;
    float absmax = 0.f, ext = 0.f;
    bool ok = true;
    for (int a = 0; a < 3; ++a) ok = ok && lo[a] <= hi[a];
    for (int a = 0; a < 3; ++a) {
        const float l = ok ? lo[a] : 0.f, h = ok ? hi[a] : 0.f;
        absmax = std::max(absmax, std::max(std::fabs(l), std::fabs(h)));
        ext = std::max(ext, h - l);
    }
    const float pad = 0x1p-14f * absmax + 1e-30f;
    for (int a = 0; a < 3; ++a) {
        b.lo[a] = (ok ? lo[a] : 0.f) - pad;
        b.hi[a] = (ok ? hi[a] : 0.f) + pad;
    }
    b.scale = std::max(absmax, ext);
    return b;
}
// the tree-related members of a traversal launch
static void trace_args_scene(TraceArgs &a, const b200pt_scene *s) {
    a.nodes = s->d_nodes;
    a.tri_base = s->d_tri_base;
    a.lut = s->d_lut;
    a.bounds = s->trav_bounds;
    a.tlas_bounds = s->tlas_bounds;
    a.tris = s->d_tris;
    a.magic = 0x47000000u;
}

extern "C" {

// ------------------------------------------------------------------- context
int b200pt_ctx_create(int device, b200pt_ctx **out) {
    if (!out) return b200pt_fail(B200PT_ERR_INVALID, "ctx_create: out is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return b200pt_fail(B200PT_ERR_NO_DEVICE, "no usable CUDA device (%s); this library has no CPU fallback",
                           e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    if (device < 0 || device >= n) return b200pt_fail(B200PT_ERR_INVALID, "ctx_create: device %d out of range", device);
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return b200pt_fail(B200PT_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device,
                           prop.major, prop.minor);
    b200pt_ctx *c = new b200pt_ctx;
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&c->stream_aux, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
    *out = c;
    return B200PT_OK;
}

void b200pt_ctx_destroy(b200pt_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->stream_aux) cudaStreamDestroy(ctx->stream_aux);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    delete ctx;
}

int b200pt_ctx_synchronize(b200pt_ctx *ctx) {
    if (!ctx) return b200pt_fail(B200PT_ERR_INVALID, "ctx is NULL");
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return B200PT_OK;
}

uint64_t b200pt_ctx_stream(b200pt_ctx *ctx) { return ctx ? (uint64_t)(uintptr_t)ctx->stream : 0; }

int b200pt_ctx_set_option(b200pt_ctx *ctx, const char *key, int64_t value) {
    if (!ctx || !key) return b200pt_fail(B200PT_ERR_INVALID, "ctx_set_option: NULL argument");
    if (!strcmp(key, "gpu_bvh_build")) {
        ctx->gpu_bvh_build = value != 0;
        return B200PT_OK;
    }
    return b200pt_fail(B200PT_ERR_INVALID, "ctx_set_option: unknown option '%s'", key);
}

// --------------------------------------------------------------------- scene
int b200pt_scene_create(b200pt_ctx *ctx, const b200pt_scene_desc *d, b200pt_scene **out) {
    if (!ctx || !d || !out) return b200pt_fail(B200PT_ERR_INVALID, "scene_create: NULL argument");
    if (d->n_triangles < 0 || (d->n_triangles > 0 && (!d->vertices || !d->material_id)))
        return b200pt_fail(B200PT_ERR_INVALID, "scene_create: vertices / material_id missing");
    if (d->n_triangles >= (1ll << 31)) return b200pt_fail(B200PT_ERR_INVALID, "scene_create: too many triangles");
    if (d->n_materials <= 0 || !d->materials) return b200pt_fail(B200PT_ERR_INVALID, "scene_create: no materials");
    if (d->n_materials > 65535) return b200pt_fail(B200PT_ERR_INVALID, "scene_create: more than 65535 materials");
    if (d->n_spectrum_samples != 0 && d->n_spectrum_samples != B200PT_SPECTRUM_SAMPLES)
        return b200pt_fail(B200PT_ERR_INVALID, "scene_create: n_spectrum_samples is %d (0 = RGBSpectrum host, %d = SampledSpectrum host)",
                           d->n_spectrum_samples, B200PT_SPECTRUM_SAMPLES);
    if (d->n_spectrum_samples != 0 && (!d->material_spectra || !d->cie_xyz || (d->n_lights > 0 && !d->light_spectra)))
        return b200pt_fail(B200PT_ERR_INVALID, "scene_create: a SampledSpectrum host must pass material_spectra, light_spectra and cie_xyz");
    for (int i = 0; i < d->n_materials; ++i)
        if (d->materials[i].type < 0 || d->materials[i].type > B200PT_MAT_GLASS)
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: material %d has unsupported type %d", i,
                               d->materials[i].type);
    for (int64_t i = 0; i < d->n_triangles; ++i) {
        if (d->material_id[i] < 0 || d->material_id[i] >= d->n_materials)
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: triangle %lld has material %d", (long long)i,
                               d->material_id[i]);
        if (d->light_id && (d->light_id[i] < -1 || d->light_id[i] >= d->n_lights))
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: triangle %lld has light %d", (long long)i,
                               d->light_id[i]);
    }
    if (d->n_spheres < 0 || (d->n_spheres > 0 && !d->spheres) || d->n_spheres > 4096)
        return b200pt_fail(B200PT_ERR_INVALID, "scene_create: bad sphere array (at most 4096 spheres; they are not in the BVH)");
    for (int i = 0; i < d->n_spheres; ++i) {
        const b200pt_sphere &sp = d->spheres[i];
        if (!(sp.radius > 0.f) || sp.material_id < 0 || sp.material_id >= d->n_materials || sp.light_id < -1 ||
            sp.light_id >= d->n_lights)
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: sphere %d has a bad radius, material or light", i);
    }
    for (int i = 0; i < d->n_lights; ++i) {
        const int kind = d->lights[i].kind;
        if (kind < B200PT_LIGHT_AREA || kind > B200PT_LIGHT_DISTANT)
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: light %d has unknown kind %d", i, kind);
        if (kind != B200PT_LIGHT_AREA) continue;  // delta lights have no geometry
        const int sph = d->lights[i].sphere;
        if (sph >= 0) {
            if (sph >= d->n_spheres || d->spheres[sph].light_id != i)
                return b200pt_fail(B200PT_ERR_INVALID, "scene_create: light %d and spheres[].light_id disagree", i);
            continue;
        }
        int t = d->lights[i].triangle;
        if (t < 0 || t >= d->n_triangles || !d->light_id || d->light_id[t] != i)
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: light %d and light_id[] disagree", i);
    }
    CUDA_TRY(cudaSetDevice(ctx->device));

    bool gpu_build = ctx->gpu_bvh_build;
    if (const char *e = getenv("B200PT_BVH_BUILD")) gpu_build = !strcmp(e, "gpu");
    if (d->n_instances > 0) gpu_build = false;  // object instances: the per-object trees come from the host builder
    // object instancing (b200pt_instance): distinct triangle ranges = objects
    if (d->n_instances < 0 || (d->n_instances > 0 && !d->instances) || d->n_instances > 65536)
        return b200pt_fail(B200PT_ERR_INVALID, "scene_create: bad instance array (at most 65536 instances)");
    const int64_t n_top = d->n_instances > 0 ? d->n_toplevel_triangles : d->n_triangles;
    if (n_top < 0 || n_top > d->n_triangles) return b200pt_fail(B200PT_ERR_INVALID, "scene_create: bad n_toplevel_triangles");
    std::vector<std::pair<int64_t, int64_t>> obj_ranges;
    std::vector<int> inst_object((size_t)d->n_instances);
    for (int i = 0; i < d->n_instances; ++i) {
        const b200pt_instance &in = d->instances[i];
        if (in.first_triangle < n_top || in.n_triangles <= 0 || in.first_triangle + in.n_triangles > d->n_triangles)
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: instance %d names triangles outside the object range", i);
        for (int64_t t = in.first_triangle; t < in.first_triangle + in.n_triangles; ++t)
            if (d->light_id && d->light_id[t] >= 0)
                return b200pt_fail(B200PT_ERR_INVALID, "scene_create: area lights cannot sit inside instances (api.cpp:1411-1413)");
        const std::pair<int64_t, int64_t> rg(in.first_triangle, in.n_triangles);
        size_t oi = std::find(obj_ranges.begin(), obj_ranges.end(), rg) - obj_ranges.begin();
        if (oi == obj_ranges.size()) obj_ranges.push_back(rg);
        inst_object[i] = (int)oi;
    }
    std::vector<uint32_t> obj_node_off(obj_ranges.size()), obj_tri_off(obj_ranges.size());
    std::vector<TravBounds> obj_bounds(obj_ranges.size());
    Wbvh bvh;
    GpuBuildOutput gout;
    uint64_t n_top_nodes = 0;
    if (gpu_build) {
        // ---- on-device build (wbvh_gpu.cu): Morton order -> binary radix tree -> 7-wide collapse
        GpuBuildInput gin;
        gin.vertices = d->vertices;
        gin.n_tris = d->n_triangles;
        gin.material_id = d->material_id;
        gin.light_id = d->light_id;
        gin.flip = d->flip_normal;
        gin.vertex_flags = d->vertex_flags;
        gin.uvs = d->uvs;
        gin.has_normals = d->normals != nullptr;
        char msg[256] = "";
        auto drop = [&]() {
            cudaFree(gout.d_nodes);
            cudaFree(gout.d_tri_base);
            cudaFree(gout.d_tris);
            cudaFree(gout.d_prim_to_tri);
        };
        if (!build_wbvh_gpu(gin, ctx->stream, &gout, msg, sizeof(msg))) {
            drop();
            return b200pt_fail(B200PT_ERR_CUDA, "scene_create: device BVH build failed: %s", msg);
        }
        if (gout.max_depth > B200PT_STACK - 4) {
            drop();
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: device-built BVH depth %d exceeds the traversal stack (use the host builder)",
                               gout.max_depth);
        }
        bvh.prim_to_tri.resize((size_t)d->n_triangles);
        cudaError_t ce = cudaMemcpy(bvh.prim_to_tri.data(), gout.d_prim_to_tri, (size_t)d->n_triangles * 4, cudaMemcpyDeviceToHost);
        cudaFree(gout.d_prim_to_tri);
        gout.d_prim_to_tri = nullptr;
        if (ce != cudaSuccess) {
            drop();
            return b200pt_fail(B200PT_ERR_CUDA, "scene_create: prim_to_tri download failed: %s", cudaGetErrorString(ce));
        }
    } else {
    // triangles the reference can never hit (shapes/triangle.cpp:304-312)
    std::vector<uint8_t> degenerate((size_t)d->n_triangles);
    for (int64_t i = 0; i < d->n_triangles; ++i) {
        const float *v = d->vertices + 9 * i;
        V3 dpdu, dpdv;
        TriShading sh;
        default_shading(&sh);
        const uint8_t vf = d->vertex_flags ? d->vertex_flags[i] : 3;
        if (d->uvs && (vf & 2)) memcpy(sh.uv, d->uvs + 6 * i, sizeof(float) * 6);
        degenerate[i] = !triangle_partials(mk(v[0], v[1], v[2]), mk(v[3], v[4], v[5]), mk(v[6], v[7], v[8]), sh.uv, &dpdu, &dpdv);
    }
    int threads = (int)std::thread::hardware_concurrency();
    if (const char *e = getenv("B200PT_BUILD_THREADS")) threads = atoi(e);
    build_wbvh(d->vertices, n_top, d->material_id, d->light_id, d->flip_normal, degenerate.data(), std::max(1, threads), &bvh);
    if (bvh.max_depth > B200PT_STACK - 4)
        return b200pt_fail(B200PT_ERR_INVALID, "scene_create: BVH depth %d exceeds the traversal stack", bvh.max_depth);
    {
        int64_t bad = validate_wbvh(bvh);
        if (bad) return b200pt_fail(B200PT_ERR_INVALID, "scene_create: BVH validation found %lld violations", (long long)bad);
    }
    n_top_nodes = bvh.nodes.size();
    // one tree per object, appended behind the top-level one; k_spheres traverses them through offset pointers,
    // so their node / triangle indices stay relative to the object's own arrays
    bvh.prim_to_tri.resize((size_t)d->n_triangles, 0xffffffffu);
    for (size_t o = 0; o < obj_ranges.size(); ++o) {
        const int64_t first = obj_ranges[o].first, count = obj_ranges[o].second;
        Wbvh ob;
        build_wbvh(d->vertices + 9 * first, count, d->material_id + first, d->light_id ? d->light_id + first : nullptr,
                   d->flip_normal ? d->flip_normal + first : nullptr, degenerate.data() + first, std::max(1, threads), &ob);
        if (ob.max_depth > B200PT_STACK - 4)
            return b200pt_fail(B200PT_ERR_INVALID, "scene_create: BVH depth %d of an object exceeds the traversal stack", ob.max_depth);
        const int64_t bad = validate_wbvh(ob);
        if (bad) return b200pt_fail(B200PT_ERR_INVALID, "scene_create: object BVH validation found %lld violations", (long long)bad);
        obj_node_off[o] = (uint32_t)bvh.nodes.size();
        obj_tri_off[o] = (uint32_t)bvh.tris.size();
        bvh.nodes.insert(bvh.nodes.end(), ob.nodes.begin(), ob.nodes.end());
        bvh.tri_base.insert(bvh.tri_base.end(), ob.tri_base.begin(), ob.tri_base.end());
        obj_bounds[o] = make_trav_bounds(ob.bounds_lo, ob.bounds_hi);
        for (TriRecord t : ob.tris) {
            t.prim += (uint32_t)first;      // back to the scene's triangle numbering
            t.mat_flags |= 0x100000u;       // object-space triangle: shading goes through the instance transform
            bvh.tris.push_back(t);
        }
        for (int64_t i = 0; i < count; ++i) bvh.prim_to_tri[(size_t)(first + i)] = obj_tri_off[o] + ob.prim_to_tri[(size_t)i];
    }
    // triangles of objects that no instance uses still need records (prim_to_tri must be total)
    for (int64_t i = n_top; i < d->n_triangles; ++i)
        if (bvh.prim_to_tri[(size_t)i] == 0xffffffffu) {
            TriRecord t;
            memset(&t, 0, sizeof(t));
            const float *v = d->vertices + 9 * i;
            memcpy(t.p0, v, 12);
            memcpy(t.p1, v + 3, 12);
            memcpy(t.p2, v + 6, 12);
            t.prim = (uint32_t)i;
            t.mat_flags = (uint32_t)d->material_id[i] | 0x20000u | 0x100000u;
            t.light = -1;
            bvh.prim_to_tri[(size_t)i] = (uint32_t)bvh.tris.size();
            bvh.tris.push_back(t);
        }
    }
    std::vector<DevInstance> dinst((size_t)d->n_instances);
    for (int i = 0; i < d->n_instances; ++i) {
        const b200pt_instance &in = d->instances[i];
        DevInstance &di = dinst[i];
        memcpy(di.i2w, in.instance_to_world, sizeof(di.i2w));
        memcpy(di.w2i, in.world_to_instance, sizeof(di.w2i));
        di.is_identity = in.is_identity != 0;
        di.node_off = obj_node_off[inst_object[i]];
        di.tri_off = obj_tri_off[inst_object[i]];
        for (int a = 0; a < 3; ++a) {
            di.obj_lo[a] = obj_bounds[inst_object[i]].lo[a];
            di.obj_hi[a] = obj_bounds[inst_object[i]].hi[a];
        }
        di.obj_scale = obj_bounds[inst_object[i]].scale;
        // TransformedPrimitive::WorldBound (primitive.h:104-106): InstanceToWorld(bounds of the object), 8 corners
        float olo[3] = {INFINITY, INFINITY, INFINITY}, ohi[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int64_t v = 3 * in.first_triangle; v < 3 * (in.first_triangle + in.n_triangles); ++v)
            for (int a = 0; a < 3; ++a) {
                olo[a] = std::min(olo[a], d->vertices[3 * v + a]);
                ohi[a] = std::max(ohi[a], d->vertices[3 * v + a]);
            }
        float wlo[3] = {INFINITY, INFINITY, INFINITY}, whi[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int c = 0; c < 8; ++c) {
            const V3 q = xform_point(di.i2w, mk((c & 1) ? ohi[0] : olo[0], (c & 2) ? ohi[1] : olo[1], (c & 4) ? ohi[2] : olo[2]));
            for (int a = 0; a < 3; ++a) {
                wlo[a] = std::min(wlo[a], comp(q, a));
                whi[a] = std::max(whi[a], comp(q, a));
            }
        }
        bool unset = true;
        for (int a = 0; a < 6; ++a) unset = unset && in.leaf_bounds[a] == 0.f;
        for (int a = 0; a < 3; ++a) {
            di.leaf_lo[a] = unset ? wlo[a] : in.leaf_bounds[a];
            di.leaf_hi[a] = unset ? whi[a] : in.leaf_bounds[3 + a];
            di.world_lo[a] = wlo[a];
            di.world_hi[a] = whi[a];
        }
    }
    // a tree over the instances' leaf boxes (each box enters the builder as a triangle spanning it; the leaf
    // "triangles" of this tree carry instance numbers and are only ever read by k_spheres): scenes with many instances
    uint32_t tlas_node_off = 0, tlas_tri_off = 0;
    const float zero3[3] = {0.f, 0.f, 0.f};
    TravBounds tlas_bounds = make_trav_bounds(zero3, zero3);
    if (d->n_instances > 0 && !gpu_build) {
        std::vector<float> boxes((size_t)d->n_instances * 9);
        std::vector<int32_t> zeros((size_t)d->n_instances, 0);
        for (int i = 0; i < d->n_instances; ++i) {
            const DevInstance &di = dinst[i];
            float *v = boxes.data() + 9 * (size_t)i;
            v[0] = di.leaf_lo[0], v[1] = di.leaf_lo[1], v[2] = di.leaf_lo[2];
            v[3] = di.leaf_hi[0], v[4] = di.leaf_hi[1], v[5] = di.leaf_hi[2];
            v[6] = di.leaf_lo[0], v[7] = di.leaf_hi[1], v[8] = di.leaf_lo[2];
        }
        Wbvh tl;
        build_wbvh(boxes.data(), d->n_instances, zeros.data(), nullptr, nullptr, nullptr, 1, &tl);
        if (tl.max_depth <= B200PT_STACK - 4 && validate_wbvh(tl) == 0 && tl.n_in_leaves == (uint32_t)d->n_instances) {
            tlas_node_off = (uint32_t)bvh.nodes.size();
            tlas_tri_off = (uint32_t)bvh.tris.size();
            bvh.nodes.insert(bvh.nodes.end(), tl.nodes.begin(), tl.nodes.end());
            bvh.tri_base.insert(bvh.tri_base.end(), tl.tri_base.begin(), tl.tri_base.end());
            bvh.tris.insert(bvh.tris.end(), tl.tris.begin(), tl.tris.end());
            tlas_bounds = make_trav_bounds(tl.bounds_lo, tl.bounds_hi);
        }
    }

    const size_t n_tri_records = gpu_build ? (size_t)gout.n_tris : bvh.tris.size();
    const size_t n_node_records = gpu_build ? (size_t)gout.n_nodes : bvh.nodes.size();
    // per-vertex shading data in leaf order + flags (bit 18 normals, bit 19 uvs) in the triangle records
    std::vector<F4> tri_n, tri_uv;
    if (d->normals) tri_n.assign(n_tri_records * 3, F4{0, 0, 0, 0});
    if (d->uvs) tri_uv.assign(n_tri_records * 2, F4{0, 0, 0, 0});
    for (int64_t i = 0; i < d->n_triangles; ++i) {
        const uint8_t vf = d->vertex_flags ? d->vertex_flags[i] : 3;
        const uint32_t ti = bvh.prim_to_tri[i];
        if (d->normals && (vf & 1)) {
            const float *n = d->normals + 9 * i;
            for (int k = 0; k < 3; ++k) tri_n[(size_t)ti * 3 + k] = F4{n[3 * k], n[3 * k + 1], n[3 * k + 2], 0.f};
            if (!gpu_build) bvh.tris[ti].mat_flags |= 0x40000u;  // the device builder sets the flags itself
        }
        if (d->uvs && (vf & 2)) {
            const float *u = d->uvs + 6 * i;
            tri_uv[(size_t)ti * 2] = F4{u[0], u[1], u[2], u[3]};
            tri_uv[(size_t)ti * 2 + 1] = F4{u[4], u[5], 0.f, 0.f};
            if (!gpu_build) bvh.tris[ti].mat_flags |= 0x80000u;
        }
    }

    b200pt_scene *s = new b200pt_scene;
    s->ctx = ctx;
    s->n_nodes = n_node_records;
    s->n_top_nodes = gpu_build ? (uint64_t)gout.n_nodes : n_top_nodes;
    s->n_tris = n_tri_records;
    s->materials.assign(d->materials, d->materials + d->n_materials);
    s->lights.assign(d->lights, d->lights + d->n_lights);
    s->nspec = d->n_spectrum_samples;
    if (s->nspec) {
        const size_t ns = (size_t)s->nspec;
        s->material_spectra.assign(d->material_spectra, d->material_spectra + (size_t)d->n_materials * B200PT_MATERIAL_SPECTRA * ns);
        if (d->n_lights > 0) s->light_spectra.assign(d->light_spectra, d->light_spectra + (size_t)d->n_lights * ns);
        s->cie_xyz.assign(d->cie_xyz, d->cie_xyz + 3 * ns);
    }
    s->prim_to_tri = std::move(bvh.prim_to_tri);
    for (int a = 0; a < 3; ++a) {
        s->bounds_lo[a] = INFINITY;
        s->bounds_hi[a] = -INFINITY;
    }
    for (int64_t i = 0; i < 3 * n_top; ++i)  // object triangles enter through their instances' bounds
        for (int a = 0; a < 3; ++a) {
            const float v = d->vertices[3 * i + a];
            if (std::isfinite(v)) {
                s->bounds_lo[a] = std::min(s->bounds_lo[a], v);
                s->bounds_hi[a] = std::max(s->bounds_hi[a], v);
            }
        }
    s->n_prims = (uint64_t)d->n_triangles;
    s->spheres.resize((size_t)d->n_spheres);
    for (int i = 0; i < d->n_spheres; ++i) {
        const b200pt_sphere &in = d->spheres[i];
        DevSphere &sp = s->spheres[i];
        memcpy(sp.o2w, in.object_to_world, sizeof(sp.o2w));
        memcpy(sp.w2o, in.world_to_object, sizeof(sp.w2o));
        // Sphere ctor (sphere.h:49-61): a full sphere (zMin = -r, zMax = r, phiMax = Radians(360)) unless the host
        // passed the members of a clipped one
        const float r = in.radius;
        sp.radius = r;
        float zMin = pt_clamp(pt_min(-r, r), -r, r), zMax = pt_clamp(pt_max(-r, r), -r, r);
        sp.theta_min = pt_acosf(pt_clamp(pt_min(zMin, zMax) / r, -1.f, 1.f));
        sp.theta_max = pt_acosf(pt_clamp(pt_max(zMin, zMax) / r, -1.f, 1.f));
        sp.phi_max = (PT_PI / 180) * pt_clamp(360.f, 0.f, 360.f);
        if (in.phi_max != 0.f) {
            zMin = in.z_min;
            zMax = in.z_max;
            sp.theta_min = in.theta_min;
            sp.theta_max = in.theta_max;
            sp.phi_max = in.phi_max;
        }
        sp.z_min = zMin;
        sp.z_max = zMax;
        sp.area = sp.phi_max * r * (zMax - zMin);
        const bool flip = (in.reverse_orientation != 0) ^ (in.transform_swaps_handedness != 0);
        sp.mat_flags = (uint32_t)in.material_id | (flip ? 0x10000u : 0u);
        sp.light_id = in.light_id;
        sp.reverse_orientation = in.reverse_orientation != 0;
        // Shape::WorldBound (shape.cpp:52, transform.cpp:246-256) joins Scene::WorldBound()
        float wlo[3] = {INFINITY, INFINITY, INFINITY}, whi[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int c = 0; c < 8; ++c) {
            const V3 q = xform_point(sp.o2w, mk((c & 1) ? r : -r, (c & 2) ? r : -r, (c & 4) ? zMax : zMin));  // ObjectBound
            for (int a = 0; a < 3; ++a) {
                wlo[a] = std::min(wlo[a], comp(q, a));
                whi[a] = std::max(whi[a], comp(q, a));
                s->bounds_lo[a] = std::min(s->bounds_lo[a], comp(q, a));
                s->bounds_hi[a] = std::max(s->bounds_hi[a], comp(q, a));
            }
        }
        bool unset = true;
        for (int a = 0; a < 6; ++a) unset = unset && in.leaf_bounds[a] == 0.f;
        for (int a = 0; a < 3; ++a) {
            sp.leaf_lo[a] = unset ? wlo[a] : in.leaf_bounds[a];
            sp.leaf_hi[a] = unset ? whi[a] : in.leaf_bounds[3 + a];
        }
    }
    s->instances = dinst;
    s->tlas_node_off = tlas_node_off;
    s->tlas_tri_off = tlas_tri_off;
    s->tlas_bounds = tlas_bounds;
    s->trav_bounds = gpu_build ? make_trav_bounds(gout.bounds_lo, gout.bounds_hi) : make_trav_bounds(bvh.bounds_lo, bvh.bounds_hi);
    for (const DevInstance &di : dinst)  // TransformedPrimitive::WorldBound joins Scene::WorldBound()
        for (int a = 0; a < 3; ++a) {
            s->bounds_lo[a] = std::min(s->bounds_lo[a], di.world_lo[a]);
            s->bounds_hi[a] = std::max(s->bounds_hi[a], di.world_hi[a]);
        }
    s->light_area.resize(d->n_lights);
    for (int i = 0; i < d->n_lights; ++i) {
        if (d->lights[i].kind != B200PT_LIGHT_AREA) {
            s->light_area[i] = 0.f;
            continue;
        }
        if (d->lights[i].sphere >= 0) {
            s->light_area[i] = s->spheres[d->lights[i].sphere].area;
            continue;
        }
        const float *v = d->vertices + 9 * (int64_t)d->lights[i].triangle;
        s->light_area[i] = triangle_area(mk(v[0], v[1], v[2]), mk(v[3], v[4], v[5]), mk(v[6], v[7], v[8]));
    }
    cudaError_t e;
    if (gpu_build) {
        s->d_nodes = static_cast<U4 *>(gout.d_nodes);
        s->d_tri_base = static_cast<uint32_t *>(gout.d_tri_base);
        s->d_tris = static_cast<F4 *>(gout.d_tris);
    }
    if ((!gpu_build && ((e = cudaMalloc(&s->d_nodes, std::max<size_t>(1, n_node_records) * sizeof(WbvhNode))) != cudaSuccess ||
                        (e = cudaMalloc(&s->d_tri_base, std::max<size_t>(1, n_node_records) * sizeof(uint32_t))) != cudaSuccess ||
                        (e = cudaMalloc(&s->d_tris, std::max<size_t>(1, n_tri_records) * sizeof(TriRecord))) != cudaSuccess)) ||
        (e = cudaMalloc(&s->d_materials, s->materials.size() * sizeof(b200pt_material))) != cudaSuccess ||
        (e = cudaMalloc(&s->d_material_spectra, std::max<size_t>(1, s->material_spectra.size()) * sizeof(float))) != cudaSuccess ||
        (e = cudaMalloc(&s->d_spheres, std::max<size_t>(1, s->spheres.size()) * sizeof(DevSphere))) != cudaSuccess ||
        (e = cudaMalloc(&s->d_instances, std::max<size_t>(1, s->instances.size()) * sizeof(DevInstance))) != cudaSuccess ||
        (e = cudaMalloc(&s->d_lut, B200PT_LUT_BYTES)) != cudaSuccess ||
        (e = cudaMalloc(&s->d_work, 64)) != cudaSuccess) {
        b200pt_scene_destroy(s);
        return b200pt_fail(B200PT_ERR_OOM, "scene_create: cudaMalloc failed: %s", cudaGetErrorString(e));
    }
    if ((e = cudaMallocHost(&s->h_nodes, std::max<size_t>(1, n_node_records) * sizeof(WbvhNode))) != cudaSuccess ||
        (e = cudaMallocHost(&s->h_tri_base, std::max<size_t>(1, n_node_records) * sizeof(uint32_t))) != cudaSuccess ||
        (e = cudaMallocHost(&s->h_tris, std::max<size_t>(1, n_tri_records) * sizeof(TriRecord))) != cudaSuccess) {
        b200pt_scene_destroy(s);
        return b200pt_fail(B200PT_ERR_OOM, "scene_create: cudaMallocHost failed: %s", cudaGetErrorString(e));
    }
    if (!tri_n.empty()) {
        if ((e = cudaMalloc(&s->d_tri_n, tri_n.size() * sizeof(F4))) != cudaSuccess ||
            (e = cudaMemcpy(s->d_tri_n, tri_n.data(), tri_n.size() * sizeof(F4), cudaMemcpyHostToDevice)) != cudaSuccess) {
            b200pt_scene_destroy(s);
            return b200pt_fail(B200PT_ERR_OOM, "scene_create: shading normals upload failed: %s", cudaGetErrorString(e));
        }
    }
    if (!tri_uv.empty()) {
        if ((e = cudaMalloc(&s->d_tri_uv, tri_uv.size() * sizeof(F4))) != cudaSuccess ||
            (e = cudaMemcpy(s->d_tri_uv, tri_uv.data(), tri_uv.size() * sizeof(F4), cudaMemcpyHostToDevice)) != cudaSuccess) {
            b200pt_scene_destroy(s);
            return b200pt_fail(B200PT_ERR_OOM, "scene_create: uv upload failed: %s", cudaGetErrorString(e));
        }
    }
    if (gpu_build) {
        // keep host copies like the host path does (b200pt_scene_upload re-sends them; B200PT_VALIDATE_BVH checks them)
        if ((e = cudaMemcpy(s->h_nodes, s->d_nodes, n_node_records * sizeof(WbvhNode), cudaMemcpyDeviceToHost)) != cudaSuccess ||
            (e = cudaMemcpy(s->h_tri_base, s->d_tri_base, n_node_records * sizeof(uint32_t), cudaMemcpyDeviceToHost)) != cudaSuccess ||
            (e = cudaMemcpy(s->h_tris, s->d_tris, n_tri_records * sizeof(TriRecord), cudaMemcpyDeviceToHost)) != cudaSuccess) {
            b200pt_scene_destroy(s);
            return b200pt_fail(B200PT_ERR_CUDA, "scene_create: BVH download failed: %s", cudaGetErrorString(e));
        }
        if (getenv("B200PT_VALIDATE_BVH")) {
            Wbvh chk;
            chk.nodes.assign(static_cast<WbvhNode *>(s->h_nodes), static_cast<WbvhNode *>(s->h_nodes) + n_node_records);
            chk.tri_base.assign(static_cast<uint32_t *>(s->h_tri_base), static_cast<uint32_t *>(s->h_tri_base) + n_node_records);
            chk.tris.assign(static_cast<TriRecord *>(s->h_tris), static_cast<TriRecord *>(s->h_tris) + n_tri_records);
            chk.prim_to_tri = s->prim_to_tri;
            chk.n_in_leaves = gout.n_in_leaves;
            chk.max_depth = gout.max_depth;
            const int64_t bad = validate_wbvh(chk);
            if (bad) {
                b200pt_scene_destroy(s);
                return b200pt_fail(B200PT_ERR_INVALID, "scene_create: device-built BVH failed validation (%lld violations)", (long long)bad);
            }
        }
    } else {
        memcpy(s->h_nodes, bvh.nodes.data(), bvh.nodes.size() * sizeof(WbvhNode));
        memcpy(s->h_tri_base, bvh.tri_base.data(), bvh.tri_base.size() * sizeof(uint32_t));
        memcpy(s->h_tris, bvh.tris.data(), bvh.tris.size() * sizeof(TriRecord));
    }
    int rc = b200pt_scene_upload(s, nullptr);
    if (rc != B200PT_OK) {
        b200pt_scene_destroy(s);
        return rc;
    }
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *out = s;
    return B200PT_OK;
}

int b200pt_scene_upload(b200pt_scene *s, uint64_t *bytes) {
    if (!s) return b200pt_fail(B200PT_ERR_INVALID, "scene is NULL");
    CUDA_TRY(cudaSetDevice(s->ctx->device));
    cudaStream_t st = s->ctx->stream;
    const size_t nb = s->n_nodes * sizeof(WbvhNode), tb = s->n_tris * sizeof(TriRecord),
                 mb = s->materials.size() * sizeof(b200pt_material), bb = s->n_nodes * sizeof(uint32_t);
    CUDA_TRY(cudaMemcpyAsync(s->d_nodes, s->h_nodes, nb, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(s->d_tri_base, s->h_tri_base, bb, cudaMemcpyHostToDevice, st));
    {
        static uint8_t lut[B200PT_LUT_BYTES];  // the same table for every scene
        for (uint32_t o = 0; o < 8; ++o)
            for (uint32_t m = 0; m < 256; ++m) lut[o << 8 | m] = (uint8_t)permute_slots(m, o);
        CUDA_TRY(cudaMemcpyAsync(s->d_lut, lut, sizeof(lut), cudaMemcpyHostToDevice, st));
    }
    CUDA_TRY(cudaMemcpyAsync(s->d_tris, s->h_tris, tb, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(s->d_materials, s->materials.data(), mb, cudaMemcpyHostToDevice, st));
    const size_t msb = s->material_spectra.size() * sizeof(float);
    if (msb) CUDA_TRY(cudaMemcpyAsync(s->d_material_spectra, s->material_spectra.data(), msb, cudaMemcpyHostToDevice, st));
    const size_t sb = s->spheres.size() * sizeof(DevSphere);
    if (sb) CUDA_TRY(cudaMemcpyAsync(s->d_spheres, s->spheres.data(), sb, cudaMemcpyHostToDevice, st));
    const size_t ib = s->instances.size() * sizeof(DevInstance);
    if (ib) CUDA_TRY(cudaMemcpyAsync(s->d_instances, s->instances.data(), ib, cudaMemcpyHostToDevice, st));
    if (bytes) *bytes = nb + bb + tb + mb + sb + ib + msb + B200PT_LUT_BYTES;
    return B200PT_OK;
}

void b200pt_scene_destroy(b200pt_scene *s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    cudaFree(s->d_nodes);
    cudaFree(s->d_tri_base);
    cudaFree(s->d_lut);
    cudaFree(s->d_tris);
    cudaFree(s->d_materials);
    cudaFree(s->d_material_spectra);
    cudaFree(s->d_tri_n);
    cudaFree(s->d_tri_uv);
    cudaFree(s->d_spheres);
    cudaFree(s->d_instances);
    cudaFree(s->d_work);
    cudaFreeHost(s->h_nodes);
    cudaFreeHost(s->h_tri_base);
    cudaFreeHost(s->h_tris);
    delete s;
}

int b200pt_scene_info(const b200pt_scene *s, uint64_t *node_bytes, uint64_t *tri_bytes, uint64_t *n_nodes) {
    if (!s) return b200pt_fail(B200PT_ERR_INVALID, "scene is NULL");
    if (node_bytes) *node_bytes = s->n_nodes * (sizeof(WbvhNode) + sizeof(uint32_t));
    if (tri_bytes) *tri_bytes = s->n_tris * sizeof(TriRecord);
    if (n_nodes) *n_nodes = s->n_nodes;
    return B200PT_OK;
}

// ------------------------------------------------- ray-batch entry points
static int trace_grid(const b200pt_ctx *ctx) { return ctx->sm_count; }  // launch_trace multiplies by its CTAs per SM
static int postpone_pct() {
    static int v = getenv("B200PT_POSTPONE_PCT") ? atoi(getenv("B200PT_POSTPONE_PCT")) : 40;
    return v;
}
static int refill_lanes() {
    static int v = getenv("B200PT_REFILL_LANES") ? atoi(getenv("B200PT_REFILL_LANES")) : 26;
    return v;
}
static int sphere_refill_lanes() {
    static int v = getenv("B200PT_SPHERE_REFILL") ? atoi(getenv("B200PT_SPHERE_REFILL")) : 8;
    return v;
}
static int trace_ctas_default() {
    static int v = getenv("B200PT_TRACE_CTAS_RT") ? atoi(getenv("B200PT_TRACE_CTAS_RT")) : 0;
    return v;
}
static int stage_nodes_default() {
    static int v = getenv("B200PT_STAGE_NODES") ? atoi(getenv("B200PT_STAGE_NODES")) : 0;
    return v;
}

// Scenes with object instances: the persistent two-level kernel (k_trace2) walks top-level triangles and instances in
// one launch.  Scenes that also hold Sphere shapes (tested by the separate pass k_spheres, which needs every earlier hit's
// distance), the CPU check build and scenes without a tree over the instances keep the separate pass for both.
static bool two_level(const b200pt_scene *s) {
#ifdef B200PT_HOST_EMU
    (void)s;
    return false;
#else
    static const bool off = getenv("B200PT_NO_TRACE2") != nullptr;
    return !off && !s->instances.empty() && s->tlas_node_off != 0 && s->spheres.empty();
#endif
}

static int trace_dev(b200pt_scene *s, uint64_t rays_dev, uint64_t out_dev, int64_t n, bool any_hit) {
    if (!s) return b200pt_fail(B200PT_ERR_INVALID, "scene is NULL");
    if (n < 0 || n >= (1ll << 32)) return b200pt_fail(B200PT_ERR_INVALID, "trace: bad ray count");
    if (n == 0) return B200PT_OK;
    CUDA_TRY(cudaSetDevice(s->ctx->device));
    cudaStream_t st = s->ctx->stream;
    uint32_t hdr[3] = {0u, (uint32_t)n, 0u};  // work counter, ray count, work counter of the sphere pass
    CUDA_TRY(cudaMemcpyAsync(s->d_work, hdr, sizeof(hdr), cudaMemcpyHostToDevice, st));
    TraceArgs a;
    memset(&a, 0, sizeof(a));
    trace_args_scene(a, s);
    a.ray_o = reinterpret_cast<const float4 *>(rays_dev);
    a.ray_d = reinterpret_cast<const float4 *>(rays_dev) + 1;
    a.stride = 2;
    a.out_stride = (int)sizeof(uint8_t);  // occ_out: one byte per ray (closest hits go to full_out)
    a.t_max_from_w = 1;
    a.count = s->d_work + 1;
    a.work = s->d_work;
    a.materials = s->d_materials;
    a.refill_lanes = refill_lanes();
    a.postpone_pct = postpone_pct();
    a.ctas = trace_ctas_default();
    a.n_staged = (uint32_t)std::min<uint64_t>((uint64_t)std::max(0, stage_nodes_default()), s->n_top_nodes);
    if (any_hit)
        a.occ_out = reinterpret_cast<uint8_t *>(out_dev);
    else
        a.full_out = reinterpret_cast<b200pt_hit *>(out_dev);
    const bool tl = two_level(s);
    a.spheres = s->d_spheres;
    a.n_spheres = (uint32_t)s->spheres.size();
    a.instances = s->d_instances;
    a.n_instances = (uint32_t)s->instances.size();
    a.tlas_node_off = s->tlas_node_off;
    a.tlas_tri_off = s->tlas_tri_off;
    a.n_tris = (uint32_t)s->n_prims;
    a.sphere_work = s->d_work + 2;
    a.sphere_refill_lanes = sphere_refill_lanes();
#ifndef B200PT_HOST_EMU
    if (tl)
        launch_trace2(a, any_hit, false, trace_grid(s->ctx), st);
    else
#endif
        launch_trace(a, any_hit, false, false, trace_grid(s->ctx), st);
    if (!s->spheres.empty() || (!s->instances.empty() && !tl)) {
        if (tl) a.n_instances = 0;  // already walked
        launch_spheres(a, any_hit, false, trace_grid(s->ctx), st);
    }
    CUDA_TRY(cudaGetLastError());
    return B200PT_OK;
}

int b200pt_trace_closest_dev(b200pt_scene *s, uint64_t rays_dev, uint64_t hits_dev, int64_t n) {
    return trace_dev(s, rays_dev, hits_dev, n, false);
}
int b200pt_trace_any_dev(b200pt_scene *s, uint64_t rays_dev, uint64_t occluded_dev, int64_t n) {
    return trace_dev(s, rays_dev, occluded_dev, n, true);
}

static int trace_host(b200pt_scene *s, const b200pt_ray *rays, void *out, size_t out_elem, int64_t n, bool any_hit) {
    if (!s || (n > 0 && (!rays || !out))) return b200pt_fail(B200PT_ERR_INVALID, "trace: NULL argument");
    if (n <= 0) return n == 0 ? B200PT_OK : b200pt_fail(B200PT_ERR_INVALID, "trace: negative count");
    CUDA_TRY(cudaSetDevice(s->ctx->device));
    cudaStream_t st = s->ctx->stream;
    void *d_rays = nullptr, *d_out = nullptr;
    CUDA_TRY(cudaMalloc(&d_rays, (size_t)n * sizeof(b200pt_ray)));
    cudaError_t e = cudaMalloc(&d_out, (size_t)n * out_elem);
    if (e != cudaSuccess) {
        cudaFree(d_rays);
        return b200pt_fail(B200PT_ERR_OOM, "trace: cudaMalloc failed");
    }
    int rc = B200PT_OK;
    if (cudaMemcpyAsync(d_rays, rays, (size_t)n * sizeof(b200pt_ray), cudaMemcpyHostToDevice, st) != cudaSuccess)
        rc = b200pt_fail(B200PT_ERR_CUDA, "trace: H2D copy failed");
    if (rc == B200PT_OK) rc = trace_dev(s, (uint64_t)(uintptr_t)d_rays, (uint64_t)(uintptr_t)d_out, n, any_hit);
    if (rc == B200PT_OK && (cudaMemcpyAsync(out, d_out, (size_t)n * out_elem, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                            cudaStreamSynchronize(st) != cudaSuccess))
        rc = b200pt_fail(B200PT_ERR_CUDA, "trace: kernel or D2H copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    cudaFree(d_rays);
    cudaFree(d_out);
    return rc;
}

int b200pt_trace_closest(b200pt_scene *s, const b200pt_ray *rays, b200pt_hit *hits, int64_t n) {
    return trace_host(s, rays, hits, sizeof(b200pt_hit), n, false);
}
int b200pt_trace_any(b200pt_scene *s, const b200pt_ray *rays, uint8_t *occluded, int64_t n) {
    return trace_host(s, rays, occluded, 1, n, true);
}

}  // extern "C"

// -------------------------------------------------------------------- render
template <typename T>
static cudaError_t dev_alloc(b200pt_render *r, T **p, size_t count) {
    void *q = nullptr;
    cudaError_t e = cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) {
        r->allocs.push_back(q);
        *p = static_cast<T *>(q);
    }
    return e;
}

extern "C" {

int b200pt_render_create(b200pt_scene *scene, const b200pt_camera_desc *cam, const b200pt_film_desc *film,
                         const b200pt_sampler_desc *smp, const b200pt_integrator_desc *integ, b200pt_render **out) {
    if (!scene || !cam || !film || !smp || !integ || !out) return b200pt_fail(B200PT_ERR_INVALID, "render_create: NULL argument");
    if (!(film->filter_radius[0] > 0.f) || !(film->filter_radius[1] > 0.f) || film->filter_radius[0] > 8.f ||
        film->filter_radius[1] > 8.f)
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: pixel filter radius must be in (0, 8]");
    const bool filter_general = film->filter_table != nullptr || film->filter_radius[0] != 0.5f || film->filter_radius[1] != 0.5f;
    const bool halton = smp->type == B200PT_SAMPLER_HALTON;
    if (smp->type != B200PT_SAMPLER_SOBOL && !halton)
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: unknown sampler type %d", smp->type);
    if (smp->samples_per_pixel <= 0 || (!halton && (smp->samples_per_pixel & (smp->samples_per_pixel - 1))))
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: samples_per_pixel must be a power of two (sobol.h:52)");
    if (!halton && (!smp->matrices32 || !smp->vdc || !smp->vdc_inv || smp->n_dimensions < 5))
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: Sobol' tables missing");
    if (halton && (!smp->halton_permutations || smp->n_dimensions < 5 || smp->n_dimensions > 1000))
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: Halton permutation table missing");
    if (integ->max_depth < 0 || integ->max_depth > 200) return b200pt_fail(B200PT_ERR_INVALID, "render_create: bad max_depth");
    // 5 camera dims + per bounce: light pick 1 + uLight 2 + uScattering 2 + BSDF 2 + roulette 1
    // ... + medium channel 1 + free-flight distance 1 with VolPathIntegrator inside a medium
    const int dims_per_bounce = integ->volumetric && (integ->medium.present || integ->n_bounded_media > 0) ? 10 : 8;
    if (5 + dims_per_bounce * integ->max_depth > smp->n_dimensions)
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: max_depth %d needs %d sampler dimensions, %d provided",
                           integ->max_depth, 5 + dims_per_bounce * integ->max_depth, smp->n_dimensions);
    if (integ->medium.present && !integ->volumetric)
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: a medium needs the volumetric integrator (PathIntegrator ignores media)");
    if (integ->medium.present && scene->nspec && !integ->medium.spectra)
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: a SampledSpectrum host must pass the medium's spectra");
    if (integ->medium.present) {
        const int nb = scene->nspec ? scene->nspec : 3;
        for (int c = 0; c < nb; ++c) {
            const float sa = scene->nspec ? integ->medium.spectra[c] : integ->medium.sigma_a[c];
            const float ss = scene->nspec ? integ->medium.spectra[nb + c] : integ->medium.sigma_s[c];
            if (!(sa >= 0.f) || !(ss >= 0.f) || !(ss + sa > 0.f))
                return b200pt_fail(B200PT_ERR_INVALID, "render_create: the medium needs sigma_a, sigma_s >= 0 and sigma_t > 0 in every channel");
        }
        if (!(integ->medium.g > -1.f && integ->medium.g < 1.f))
            return b200pt_fail(B200PT_ERR_INVALID, "render_create: Henyey-Greenstein g must lie in (-1, 1)");
    }
    // media bounded by null-material spheres (ABI 6)
    const int n_bounded = integ->n_bounded_media;
    if (n_bounded < 0 || n_bounded > 4096) return b200pt_fail(B200PT_ERR_INVALID, "render_create: bad n_bounded_media");
    if (n_bounded > 0) {
        if (!integ->volumetric)
            return b200pt_fail(B200PT_ERR_INVALID, "render_create: bounded media need the volumetric integrator (PathIntegrator ignores media)");
        if (!integ->bounded_media || !integ->sphere_medium)
            return b200pt_fail(B200PT_ERR_INVALID, "render_create: bounded_media / sphere_medium missing");
        if (scene->nspec)
            return b200pt_fail(B200PT_ERR_INVALID, "render_create: bounded media are not supported for SampledSpectrum hosts");
        if (!scene->instances.empty())
            return b200pt_fail(B200PT_ERR_INVALID, "render_create: bounded media are not supported in scenes with object instances");
        for (int k = 0; k < n_bounded; ++k) {
            const b200pt_medium &m = integ->bounded_media[k];
            for (int c = 0; c < 3; ++c)
                if (!(m.sigma_a[c] >= 0.f) || !(m.sigma_s[c] >= 0.f) || !(m.sigma_a[c] + m.sigma_s[c] > 0.f))
                    return b200pt_fail(B200PT_ERR_INVALID, "render_create: bounded medium %d needs sigma_a, sigma_s >= 0 and sigma_t > 0 in every channel", k);
            if (!(m.g > -1.f && m.g < 1.f))
                return b200pt_fail(B200PT_ERR_INVALID, "render_create: bounded medium %d: Henyey-Greenstein g must lie in (-1, 1)", k);
        }
        for (size_t k = 0; k < scene->spheres.size(); ++k) {
            const int32_t mk_ = integ->sphere_medium[k];
            if (mk_ < -1 || mk_ >= n_bounded)
                return b200pt_fail(B200PT_ERR_INVALID, "render_create: sphere_medium[%zu] = %d is not a bounded medium", k, mk_);
            if (mk_ >= 0 && scene->spheres[k].light_id >= 0)
                return b200pt_fail(B200PT_ERR_INVALID, "render_create: sphere %zu bounds a medium and is an area light", k);
        }
    }
    if (integ->light_strategy != B200PT_LIGHTS_UNIFORM && integ->light_strategy != B200PT_LIGHTS_POWER &&
        integ->light_strategy != B200PT_LIGHTS_SPATIAL)
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: unsupported light sample strategy");
    const int sbw = smp->sample_bounds[2] - smp->sample_bounds[0], sbh = smp->sample_bounds[3] - smp->sample_bounds[1];
    if (sbw <= 0 || sbh <= 0) return b200pt_fail(B200PT_ERR_INVALID, "render_create: empty sample bounds");
    const int cw = film->cropped_bounds[2] - film->cropped_bounds[0], chh = film->cropped_bounds[3] - film->cropped_bounds[1];
    if (cw <= 0 || chh <= 0) return b200pt_fail(B200PT_ERR_INVALID, "render_create: empty film");

    b200pt_ctx *ctx = scene->ctx;
    CUDA_TRY(cudaSetDevice(ctx->device));
    b200pt_render *r = new b200pt_render;
    // every failure below leaves through a return: the guard frees what was allocated so far (released on success)
    struct RenderGuard {
        b200pt_render *p;
        ~RenderGuard() {
            if (p) b200pt_render_destroy(p);
        }
    } render_guard{r};
    r->scene = scene;
    r->film = *film;
    r->spp = smp->samples_per_pixel;
    RenderDev &H = r->host;
    memset(&H, 0, sizeof(H));
    H.scene.nodes = scene->d_nodes;
    H.scene.tri_base = scene->d_tri_base;
    H.scene.lut = scene->d_lut;
    H.scene.bounds = scene->trav_bounds;
    H.scene.tris = scene->d_tris;
    H.scene.materials = scene->d_materials;
    H.scene.material_spectra = scene->nspec ? scene->d_material_spectra : nullptr;
    H.scene.n_nodes = (uint32_t)scene->n_nodes;
    H.scene.n_tris = (uint32_t)scene->n_tris;
    H.scene.tri_n = scene->d_tri_n;
    H.scene.tri_uv = scene->d_tri_uv;
    H.scene.spheres = scene->d_spheres;
    H.scene.n_spheres = (uint32_t)scene->spheres.size();
    H.scene.instances = scene->d_instances;
    H.scene.n_instances = (uint32_t)scene->instances.size();
    H.scene.tlas_node_off = scene->tlas_node_off;
    H.scene.tlas_tri_off = scene->tlas_tri_off;
    // sampler (samplers/sobol.h:49-62)
    H.sampler.spp = smp->samples_per_pixel;
    memcpy(H.sampler.sb, smp->sample_bounds, sizeof(int) * 4);
    int res = 1;
    while (res < std::max(sbw, sbh)) res <<= 1;
    H.sampler.resolution = res;
    int lg = 0;
    while ((1 << lg) < res) ++lg;
    H.sampler.log2res = lg;
    H.sampler.n_dims = smp->n_dimensions;
    H.sampler.type = smp->type;
    std::vector<uint32_t> primes, prime_sums;
    if (halton) {
        // halton.cpp:74-92: scales / exponents of bases 2 and 3 covering min(extent, kMaxResolution = 128)
        const int ext[2] = {sbw, sbh};
        for (int i = 0; i < 2; ++i) {
            const int base = i == 0 ? 2 : 3;
            int scale = 1, ex = 0;
            while (scale < std::min(ext[i], 128)) {
                scale *= base;
                ++ex;
            }
            H.sampler.base_scale[i] = scale;
            H.sampler.base_exp[i] = ex;
        }
        H.sampler.sample_stride = H.sampler.base_scale[0] * H.sampler.base_scale[1];
        // multiplicativeInverse(a, n) (halton.cpp:46-63): the x in [0, n) with a*x = 1 (mod n); n <= 243 here
        auto mul_inv = [](int a, int n) {
            if (n == 1) return 0;
            for (int x = 0; x < n; ++x)
                if ((int)(((long long)a * x) % n) == 1) return x;
            return 0;
        };
        H.sampler.mult_inverse[0] = mul_inv(H.sampler.base_scale[1], H.sampler.base_scale[0]);
        H.sampler.mult_inverse[1] = mul_inv(H.sampler.base_scale[0], H.sampler.base_scale[1]);
        // Primes / PrimeSums of the bases in use (lowdiscrepancy.cpp:45-...)
        uint32_t sum = 0;
        for (uint32_t c = 2; (int)primes.size() < smp->n_dimensions; ++c) {
            bool is_prime = true;
            for (uint32_t d = 2; d * d <= c; ++d)
                if (c % d == 0) {
                    is_prime = false;
                    break;
                }
            if (!is_prime) continue;
            primes.push_back(c);
            prime_sums.push_back(sum);
            sum += c;
        }
        prime_sums.push_back(sum);
    } else {
        memcpy(H.sampler.vdc, smp->vdc, sizeof(uint64_t) * 52);
        memcpy(H.sampler.vdc_inv, smp->vdc_inv, sizeof(uint64_t) * 52);
    }
    memcpy(H.camera.r2c, cam->raster_to_camera, sizeof(float) * 16);
    memcpy(H.camera.c2w, cam->camera_to_world, sizeof(float) * 16);
    H.camera.lens_radius = cam->lens_radius;
    H.camera.focal_distance = cam->focal_distance;
    memcpy(H.crop, film->cropped_bounds, sizeof(int) * 4);
    H.filter_general = filter_general ? 1 : 0;
    for (int a = 0; a < 2; ++a) {
        H.filter_radius[a] = film->filter_radius[a];
        H.filter_inv_radius[a] = 1 / film->filter_radius[a];  // Filter::invRadius, filter.h:53-54
        // Film::GetFilmTile (film.cpp:95-106): pixels [ceil(x0 - .5 - r), floor(x1 - .5 + r) + 1)
        H.apron[a] = std::max((int)(0.f - std::ceil(0.f - 0.5f - film->filter_radius[a])),
                              (int)std::floor(0.f - 0.5f + film->filter_radius[a]) + 1);
    }
    memcpy(H.pixel_bounds, integ->pixel_bounds, sizeof(int) * 4);
    H.max_sample_luminance = film->max_sample_luminance;
    H.max_depth = integ->max_depth;
    H.rr_threshold = integ->rr_threshold;
    H.volpath = integ->volumetric ? 1 : 0;
    H.has_medium = integ->volumetric && integ->medium.present ? 1 : 0;
    for (int c = 0; c < 3 && H.has_medium; ++c) {
        H.med_sigma_s[c] = integ->medium.sigma_s[c];
        H.med_sigma_t[c] = integ->medium.sigma_s[c] + integ->medium.sigma_a[c];  // homogeneous.h:53
    }
    H.med_g = integ->medium.g;
    H.med_general = n_bounded > 0 ? 1 : 0;
    H.tiles_x = (sbw + 15) / 16;
    H.tiles_y = (sbh + 15) / 16;

    // light distribution (lightdistrib.cpp:48-82, sampling.h:57-71)
    const int nl = (int)scene->lights.size();
    std::vector<DevLight> dl(nl);
    std::vector<float> func(std::max(nl, 1), 1.f), cdf(nl + 1, 0.f);
    // DistantLight::Preprocess (distant.h:54-58): Bounds3::BoundingSphere of Scene::WorldBound() (geometry.h:808-811)
    float world_radius = 0.f;
    {
        const float *lo = scene->bounds_lo, *hi = scene->bounds_hi;
        const float inv = 1.f / 2;
        const V3 c = mk(inv * (lo[0] + hi[0]), inv * (lo[1] + hi[1]), inv * (lo[2] + hi[2]));
        const bool inside = c.x >= lo[0] && c.x <= hi[0] && c.y >= lo[1] && c.y <= hi[1] && c.z >= lo[2] && c.z <= hi[2];
        world_radius = inside ? len(c - mk(hi[0], hi[1], hi[2])) : 0.f;
    }
    bool has_delta = false;
    for (int i = 0; i < nl; ++i) {
        const b200pt_area_light &sl = scene->lights[i];
        memset(&dl[i], 0, sizeof(DevLight));
        memcpy(dl[i].lemit, sl.lemit, sizeof(float) * 3);
        dl[i].kind = sl.kind;
        if (sl.kind != B200PT_LIGHT_AREA) {
            has_delta = true;
            dl[i].tri = B200PT_MISS;
            memcpy(dl[i].position, sl.position, sizeof(float) * 3);
            dl[i].cos_total_width = sl.cos_total_width;
            dl[i].cos_falloff_start = sl.cos_falloff_start;
            memcpy(dl[i].world_to_light, sl.world_to_light, sizeof(float) * 16);
            const float wr = sl.world_radius != 0.f ? sl.world_radius : world_radius;
            dl[i].two_world_radius = 2 * wr;
            if (integ->light_strategy == B200PT_LIGHTS_POWER && nl != 1) {
                // Light::Power().y(): point.cpp:58, spot.cpp:78-80, distant.cpp:62-64 (per bin, then y())
                std::vector<float> p = host_light_spectrum(scene, i);
                for (float &c : p) {
                    if (sl.kind == B200PT_LIGHT_POINT)
                        c = (4 * PT_PI) * c;
                    else if (sl.kind == B200PT_LIGHT_SPOT)
                        c = c * 2 * PT_PI * (1 - .5f * (sl.cos_falloff_start + sl.cos_total_width));
                    else
                        c = c * PT_PI * wr * wr;
                }
                func[i] = host_spectrum_y(scene, p);
            }
            continue;
        }
        dl[i].tri = sl.sphere >= 0 ? (SPHERE_HIT_BASE | (uint32_t)sl.sphere) : scene->prim_to_tri[sl.triangle];
        dl[i].two_sided = sl.two_sided;
        dl[i].area = scene->light_area[i];
        if (integ->light_strategy == B200PT_LIGHTS_POWER && nl != 1) {
            // DiffuseAreaLight::Power().y(), diffuse.cpp:64-66 + integrator.cpp:216-224
            const float k = dl[i].two_sided ? 2.f : 1.f;
            std::vector<float> p = host_light_spectrum(scene, i);
            for (float &c : p) c = c * k * dl[i].area * PT_PI;
            func[i] = host_spectrum_y(scene, p);
        }
    }
    float funcInt = 0.f;
    if (nl > 0) {
        for (int i = 1; i < nl + 1; ++i) cdf[i] = cdf[i - 1] + func[i - 1] / nl;
        funcInt = cdf[nl];
        if (funcInt == 0) {
            for (int i = 1; i < nl + 1; ++i) cdf[i] = float(i) / float(nl);
        } else {
            for (int i = 1; i < nl + 1; ++i) cdf[i] /= funcInt;
        }
    }
    H.n_lights = nl;
    H.light_func_int = funcInt;
    // SpatialLightDistribution grid (lightdistrib.cpp:96-112, maxVoxels = 64); a single light always
    // gets the uniform distribution (lightdistrib.cpp:50)
    long long nvox = 0;
    if (integ->light_strategy == B200PT_LIGHTS_SPATIAL && nl > 1) {
        float diag[3];
        for (int a = 0; a < 3; ++a) diag[a] = scene->bounds_hi[a] - scene->bounds_lo[a];
        const int me = (diag[0] > diag[1] && diag[0] > diag[2]) ? 0 : (diag[1] > diag[2] ? 1 : 2);
        const float bmax = diag[me];
        H.grid.enabled = 1;
        for (int a = 0; a < 3; ++a) {
            H.grid.nv[a] = std::max(1, int(std::round(diag[a] / bmax * 64)));
            H.grid.wb_min[a] = scene->bounds_lo[a];
            H.grid.wb_max[a] = scene->bounds_hi[a];
        }
        nvox = (long long)H.grid.nv[0] * H.grid.nv[1] * H.grid.nv[2];
        if (nvox * (2ll * nl + 2) * 4 > (8ll << 30)) {
            return b200pt_fail(B200PT_ERR_INVALID,
                               "render_create: spatial light distribution needs %lld voxels x %d lights; use \"uniform\" or \"power\"",
                               nvox, nl);
        }
    }
    for (int a = 0; a < 3; ++a) {
        const float ext = scene->bounds_hi[a] - scene->bounds_lo[a];
        H.sort_lo[a] = scene->bounds_lo[a];
        H.sort_inv[a] = ext > 0 ? 32.f / ext : 0.f;
    }

    // batch sizing: whole tiles, about B200PT_BATCH_PATHS path slots
    // path slots per batch: 256 B of records + ~40 B of queues each, plus 5 x 60 floats with a SampledSpectrum host.
    // Larger batches keep the traversal launches fuller and spread each launch's drain over more rays: RGB takes 96 Mi slots
    // (~29 GB; cfg4 on an H100 at 400 W: +3.5 % over 32 Mi, +0.9 % over 64 Mi, profiles/README.md); 60 bins keep 16 Mi (~25 GB).
    size_t target = scene->nspec ? (16u << 20) : (96u << 20);
    if (const char *e = getenv("B200PT_BATCH_PATHS")) target = (size_t)atoll(e);
    const size_t per_tile = 256u * (size_t)r->spp;
    r->tiles_per_batch = (uint32_t)std::max<size_t>(1, target / per_tile);
    r->tiles_per_batch = std::min<uint32_t>(r->tiles_per_batch, (uint32_t)(H.tiles_x * H.tiles_y));
    const size_t cap = (size_t)r->tiles_per_batch * per_tile;
    if (cap >= (1ull << 31)) {
        return b200pt_fail(B200PT_ERR_INVALID, "render_create: one tile needs %zu path slots (too many samples)", per_tile);
    }
    H.capacity = (uint32_t)cap;

    cudaError_t e = cudaSuccess;
    uint32_t *mat32 = nullptr, *sobol_table = nullptr;
    DevLight *d_lights = nullptr;
    float *d_cdf = nullptr, *d_func = nullptr;
#define ALLOC(ptr, count) \
    if (e == cudaSuccess) e = dev_alloc(r, &(ptr), (count))
    uint16_t *d_perms = nullptr;
    uint32_t *d_primes = nullptr, *d_prime_sums = nullptr;
    if (halton) {
        ALLOC(d_perms, (size_t)prime_sums.back());
        ALLOC(d_primes, primes.size());
        ALLOC(d_prime_sums, prime_sums.size());
    } else {
        ALLOC(mat32, (size_t)smp->n_dimensions * 52);
        ALLOC(sobol_table, (size_t)smp->n_dimensions * 5 * 256);
    }
    ALLOC(d_lights, (size_t)nl);
    ALLOC(d_cdf, (size_t)nl + 1);
    ALLOC(d_func, (size_t)std::max(nl, 1));
    ALLOC(H.sp_func, (size_t)nvox * nl);
    ALLOC(H.sp_cdf, (size_t)nvox * (nl + 1));
    ALLOC(H.sp_func_int, (size_t)nvox);
    ALLOC(H.film, (size_t)cw * chh);
    ALLOC(H.path, cap);
    ALLOC(H.direct, cap);
    ALLOC(H.pix_bleed, (size_t)r->tiles_per_batch * 256);
    float *d_light_spectra = nullptr;
    if (scene->nspec) {
        const size_t spectra = cap * (size_t)scene->nspec;  // slot-major [capacity][60]
        ALLOC(H.s_beta, spectra);
        ALLOC(H.s_L, spectra);
        ALLOC(H.s_A, spectra);
        ALLOC(H.s_B, spectra);
        ALLOC(H.s_beta_ld, spectra);
        ALLOC(d_light_spectra, std::max<size_t>(1, scene->light_spectra.size()));
    }
    float *d_med_spectra = nullptr;
    std::vector<float> med_spectra;  // [sigma_s, sigma_t] of a SampledSpectrum host's medium
    if (scene->nspec && H.has_medium) {
        const int nb = scene->nspec;
        med_spectra.resize(2 * (size_t)nb);
        for (int c = 0; c < nb; ++c) {
            med_spectra[c] = integ->medium.spectra[nb + c];
            med_spectra[nb + c] = integ->medium.spectra[nb + c] + integ->medium.spectra[c];  // sigma_t(sigma_s + sigma_a)
        }
        ALLOC(d_med_spectra, med_spectra.size());
    }
    float *d_filter_table = nullptr;
    if (filter_general) {
        ALLOC(d_filter_table, 256);
        ALLOC(H.pfilm, cap);
        ALLOC(H.tile_film, (size_t)r->tiles_per_batch * (16 + 2 * H.apron[0]) * (16 + 2 * H.apron[1]));
        ALLOC(H.tile_slot, (size_t)H.tiles_x * H.tiles_y);
    }
    ALLOC(H.q_path[0], cap);
    ALLOC(H.q_path[1], cap);
    for (int m = 0; m < 4; ++m) ALLOC(H.q_mat[m], cap);
    ALLOC(H.q_shadow, cap);
    ALLOC(H.q_sorted, cap);
    ALLOC(H.sort_keys, cap);
    ALLOC(H.sort_hist, (size_t)SORT_BUCKETS);
    ALLOC(H.q_mis, cap);
    ALLOC(H.qcount, (size_t)(H.max_depth + 2) * Q_PER_BOUNCE);
    ALLOC(H.work, (size_t)(H.max_depth + 2) * 16);
    ALLOC(H.stats, 9);
    // media bounded by surfaces: medium table, per-sphere medium ids, the walkers' per-slot state
    float *d_media_tab = nullptr, *d_media_g = nullptr;
    int32_t *d_sphere_med = nullptr;
    std::vector<float> media_tab, media_g;
    std::vector<int32_t> sphere_med;
    if (H.med_general) {
        media_tab.assign((size_t)(1 + n_bounded) * 6, 0.f);
        media_g.assign((size_t)(1 + n_bounded), 0.f);
        for (int k = 0; k <= n_bounded; ++k) {
            if (k == 0 && !H.has_medium) continue;  // id 0 = the medium around the scene (never used when there is none)
            const b200pt_medium &m = k == 0 ? integ->medium : integ->bounded_media[k - 1];
            for (int c = 0; c < 3; ++c) {
                media_tab[(size_t)k * 6 + c] = m.sigma_s[c];
                media_tab[(size_t)k * 6 + 3 + c] = m.sigma_s[c] + m.sigma_a[c];  // homogeneous.h:53
            }
            media_g[(size_t)k] = m.g;
        }
        sphere_med.resize(std::max<size_t>(1, scene->spheres.size()), -1);
        for (size_t k = 0; k < scene->spheres.size(); ++k)
            sphere_med[k] = integ->sphere_medium[k] >= 0 ? integ->sphere_medium[k] + 1 : -1;
        ALLOC(d_media_tab, media_tab.size());
        ALLOC(d_media_g, media_g.size());
        ALLOC(d_sphere_med, sphere_med.size());
        ALLOC(H.cur_med, cap);
        ALLOC(H.q_cross[0], cap);
        ALLOC(H.q_cross[1], cap);
        ALLOC(H.q_walk[0], cap);
        ALLOC(H.q_walk[1], cap);
        ALLOC(H.sh_hit, cap);
        ALLOC(H.A2, cap);
        ALLOC(H.sh_tr, cap);
        ALLOC(H.mi_tr, cap);
        ALLOC(H.sh_p1, cap);
        ALLOC(H.sh_p1e, cap);
        ALLOC(H.sh_p1n, cap);
        ALLOC(r->d_walk_counts, 16);
    }
    ALLOC(r->d_dev, 1);
#undef ALLOC
    if (e != cudaSuccess) {
        return b200pt_fail(B200PT_ERR_OOM, "render_create: cudaMalloc failed: %s", cudaGetErrorString(e));
    }
    H.sampler.mat32 = mat32;
    H.sampler.table = getenv("B200PT_NO_SOBOL_TABLE") ? nullptr : sobol_table;
    H.lights = d_lights;
    H.light_spectra = d_light_spectra;
    H.med_spectra = d_med_spectra;
    H.media_tab = d_media_tab;
    H.media_g = d_media_g;
    H.sphere_med = d_sphere_med;
    H.dim_overflows = H.stats + 8;
    H.has_delta_lights = has_delta ? 1 : 0;
    H.light_cdf = d_cdf;
    H.light_func = d_func;
    cudaStream_t st = ctx->stream;
    if (halton) {
        H.sampler.perms = d_perms;
        H.sampler.primes = d_primes;
        H.sampler.prime_sums = d_prime_sums;
        CUDA_TRY(cudaMemcpyAsync(d_perms, smp->halton_permutations, (size_t)prime_sums.back() * 2, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_primes, primes.data(), primes.size() * 4, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_prime_sums, prime_sums.data(), prime_sums.size() * 4, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaStreamSynchronize(st));  // the tables above are locals / caller memory
    } else {
        CUDA_TRY(cudaMemcpyAsync(mat32, smp->matrices32, (size_t)smp->n_dimensions * 52 * 4, cudaMemcpyHostToDevice, st));
        launch_sobol_table(mat32, sobol_table, smp->n_dimensions, st);
    }
    if (nl) CUDA_TRY(cudaMemcpyAsync(d_lights, dl.data(), nl * sizeof(DevLight), cudaMemcpyHostToDevice, st));
    if (scene->nspec) {
        if (b200pt_s60::render_dev_size() != sizeof(RenderDev)) {
            return b200pt_fail(B200PT_ERR_INVALID, "render_create: the SampledSpectrum kernels were built with another RenderDev layout");
        }
        if (d_med_spectra) {
            CUDA_TRY(cudaMemcpyAsync(d_med_spectra, med_spectra.data(), med_spectra.size() * sizeof(float), cudaMemcpyHostToDevice, st));
            CUDA_TRY(cudaStreamSynchronize(st));  // med_spectra is a local
        }
        if (!scene->light_spectra.empty())
            CUDA_TRY(cudaMemcpyAsync(d_light_spectra, scene->light_spectra.data(), scene->light_spectra.size() * sizeof(float),
                                     cudaMemcpyHostToDevice, st));
        b200pt_s60::set_cie_xyz(scene->cie_xyz.data(), st);
    }
    CUDA_TRY(cudaMemcpyAsync(d_cdf, cdf.data(), (nl + 1) * sizeof(float), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(d_func, func.data(), std::max(nl, 1) * sizeof(float), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(H.film, 0, (size_t)cw * chh * sizeof(float4), st));
    if (filter_general) {
        float table[256];
        for (int i = 0; i < 256; ++i) table[i] = film->filter_table ? film->filter_table[i] : 1.f;
        H.filter_table = d_filter_table;
        CUDA_TRY(cudaMemcpyAsync(d_filter_table, table, sizeof(table), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemsetAsync(H.tile_slot, 0xff, (size_t)H.tiles_x * H.tiles_y * sizeof(int32_t), st));
        CUDA_TRY(cudaStreamSynchronize(st));  // `table` is a local
    }
    CUDA_TRY(cudaMemsetAsync(H.stats, 0, 9 * sizeof(unsigned long long), st));
    if (H.med_general) {
        CUDA_TRY(cudaMemcpyAsync(d_media_tab, media_tab.data(), media_tab.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_media_g, media_g.data(), media_g.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_sphere_med, sphere_med.data(), sphere_med.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaStreamSynchronize(st));  // locals
    }
    CUDA_TRY(cudaMemcpyAsync(r->d_dev, &H, sizeof(H), cudaMemcpyHostToDevice, st));
    if (H.grid.enabled) {
        if (scene->nspec)
            b200pt_s60::launch_spatial_build(s60(r->d_dev), s60(H), st);
        else
            launch_spatial_build(r->d_dev, H, st);
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    r->grid_trace = ctx->sm_count;  // launch_trace multiplies by its CTAs per SM
    r->grid_shade = ctx->sm_count * 8;
    // grid of the 60-bin shading kernels in CTAs per SM (B200PT_S60_SHADE_CTAS; a knob from the time they kept their
    // spectra in multi-KB local-memory frames -- with lazy spectra the frame is about 1 KB)
    r->grid_shade_s60 = ctx->sm_count * (getenv("B200PT_S60_SHADE_CTAS") ? std::max(1, atoi(getenv("B200PT_S60_SHADE_CTAS"))) : 8);
    if (getenv("B200PT_INSTRUMENT")) r->instrumented = atoi(getenv("B200PT_INSTRUMENT")) != 0;
    if (getenv("B200PT_PROFILE")) r->profiling = atoi(getenv("B200PT_PROFILE")) != 0;
    if (getenv("B200PT_SORT_FROM")) r->sort_from_bounce = atoi(getenv("B200PT_SORT_FROM"));
    if (getenv("B200PT_OVERLAP")) r->overlap = atoi(getenv("B200PT_OVERLAP")) != 0;
    r->refill_lanes = refill_lanes();
    r->postpone_pct = postpone_pct();
    r->trace_ctas = trace_ctas_default();
    r->stage_nodes = stage_nodes_default();
    render_guard.p = nullptr;
    *out = r;
    return B200PT_OK;
}

void b200pt_render_destroy(b200pt_render *r) {
    if (!r) return;
    cudaSetDevice(r->scene->ctx->device);
    cudaStreamSynchronize(r->scene->ctx->stream);
    for (void *p : r->allocs) cudaFree(p);
    cudaFree(r->d_tile_list);
    for (auto &t : r->timed) {
        cudaEventDestroy(t.a);
        cudaEventDestroy(t.b);
    }
    for (auto ev : r->event_pool) cudaEventDestroy(ev);
    delete r;
}

int b200pt_render_tile_counts(const b200pt_render *r, int32_t *nx, int32_t *ny) {
    if (!r) return b200pt_fail(B200PT_ERR_INVALID, "render is NULL");
    if (nx) *nx = r->host.tiles_x;
    if (ny) *ny = r->host.tiles_y;
    return B200PT_OK;
}

int b200pt_film_clear(b200pt_render *r) {
    if (!r) return b200pt_fail(B200PT_ERR_INVALID, "render is NULL");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    const size_t n = (size_t)(r->host.crop[2] - r->host.crop[0]) * (r->host.crop[3] - r->host.crop[1]);
    CUDA_TRY(cudaMemsetAsync(r->host.film, 0, n * sizeof(float4), r->scene->ctx->stream));
    return B200PT_OK;
}

static cudaEvent_t take_event(b200pt_render *r) {
    if (!r->event_pool.empty()) {
        cudaEvent_t e = r->event_pool.back();
        r->event_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}

struct LaunchTimer {
    b200pt_render *r;
    cudaStream_t st;
    TimedLaunch t;
    bool on;
    LaunchTimer(b200pt_render *r, cudaStream_t st, int category) : r(r), st(st), on(r->profiling) {
        r->launches++;
        r->launches_cat[category]++;
        if (on) {
            t.category = category;
            t.a = take_event(r);
            t.b = take_event(r);
            cudaEventRecord(t.a, st);
        }
    }
    ~LaunchTimer() {
        if (on) {
            cudaEventRecord(t.b, st);
            r->timed.push_back(t);
        }
    }
};

static void drain_timers(b200pt_render *r) {
    for (auto &t : r->timed) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) r->ms[t.category] += ms;
        r->event_pool.push_back(t.a);
        r->event_pool.push_back(t.b);
    }
    r->timed.clear();
}

int b200pt_render_tiles(b200pt_render *r, const int32_t *tiles, int64_t n_tiles) {
    if (!r) return b200pt_fail(B200PT_ERR_INVALID, "render is NULL");
    const int64_t total = (int64_t)r->host.tiles_x * r->host.tiles_y;
    if (n_tiles < 0 || n_tiles > (1 << 30)) return b200pt_fail(B200PT_ERR_INVALID, "render_tiles: bad tile count");
    if (!tiles && n_tiles > total) return b200pt_fail(B200PT_ERR_INVALID, "render_tiles: more tiles than the film has");
    if (n_tiles == 0) return B200PT_OK;
    b200pt_ctx *ctx = r->scene->ctx;
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    std::vector<int32_t> list((size_t)n_tiles);
    for (int64_t i = 0; i < n_tiles; ++i) {
        list[i] = tiles ? tiles[i] : (int32_t)i;
        if (list[i] < 0 || list[i] >= total) return b200pt_fail(B200PT_ERR_INVALID, "render_tiles: tile %d out of range", list[i]);
    }
    if ((size_t)n_tiles > r->tile_list_capacity) {
        CUDA_TRY(cudaStreamSynchronize(st));
        cudaFree(r->d_tile_list);
        r->d_tile_list = nullptr;
        CUDA_TRY(cudaMalloc(&r->d_tile_list, (size_t)n_tiles * sizeof(int32_t)));
        r->tile_list_capacity = (size_t)n_tiles;
    }
    // the list is consumed asynchronously: copy from a pageable vector is staged by the driver before returning
    CUDA_TRY(cudaMemcpyAsync(r->d_tile_list, list.data(), (size_t)n_tiles * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (r->host.tile_list != r->d_tile_list) {
        r->host.tile_list = r->d_tile_list;
        CUDA_TRY(cudaMemcpyAsync(r->d_dev, &r->host, sizeof(RenderDev), cudaMemcpyHostToDevice, st));
    }
    const RenderDev &H = r->host;
    const bool spectral = r->scene->nspec != 0;
    const int maxDepth = H.max_depth;
    const size_t qbytes = (size_t)(maxDepth + 2) * Q_PER_BOUNCE * sizeof(uint32_t);
    const size_t wbytes = (size_t)(maxDepth + 2) * 16 * sizeof(uint32_t);
    bool families[4] = {false, false, false, false};
    for (const auto &m : r->scene->materials) families[m.type] = true;

    for (int64_t first = 0; first < n_tiles; first += r->tiles_per_batch) {
        const uint32_t nb = (uint32_t)std::min<int64_t>(r->tiles_per_batch, n_tiles - first);
        const uint32_t n_slots = nb * 256u * (uint32_t)r->spp;
        CUDA_TRY(cudaMemsetAsync(H.qcount, 0, qbytes, st));
        CUDA_TRY(cudaMemsetAsync(H.work, 0, wbytes, st));
        CUDA_TRY(cudaMemsetAsync(H.pix_bleed, 0, (size_t)nb * 256, st));
        {
            LaunchTimer lt(r, st, 2);
            if (spectral)
                b200pt_s60::launch_raygen(s60(r->d_dev), (uint32_t)first, nb, n_slots, st);
            else
                launch_raygen(r->d_dev, (uint32_t)first, nb, n_slots, st);
        }
        // Launch order per bounce b (path.cpp:81-188):
        //   closest(b) -> shade(b) -> { any(b), MIS-closest(b) } || closest(b+1) -> resolve(b) -> shade(b+1) ...
        // The shadow / MIS rays of bounce b and the path rays of bounce b+1 are independent, so they run on
        // two streams: as the persistent CTAs of one launch drain, the other launch fills the freed SMs.
        const bool general = H.med_general != 0;  // media bounded by surfaces: boundary passes inside a bounce (see RenderDev)
        const bool medium = H.has_medium != 0 || general;  // k_medium also queues direct-lighting rays: no overlap of bounces then
        uint32_t *const wc = r->d_walk_counts;  // [0], [1] crossers of a pass (ping-pong), [2] walk kernel, [3] trace, [4] sphere pass
        auto device_count = [&](const uint32_t *d, cudaStream_t s_) {
            uint32_t v = 0;
            if (cudaMemcpyAsync(&v, d, sizeof(v), cudaMemcpyDeviceToHost, s_) != cudaSuccess) return 0u;
            if (cudaStreamSynchronize(s_) != cudaSuccess) return 0u;
            return v;
        };
        const bool overlap = r->overlap && r->sort_from_bounce < 0 && !medium;
        cudaStream_t st2 = overlap ? ctx->stream_aux : st;
        const bool tl = two_level(r->scene) && !r->instrumented;  // instances inside the traversal kernel
        const bool has_spheres = H.scene.n_spheres > 0 || (H.scene.n_instances > 0 && !tl);  // "extra shapes" pass needed
        const bool full_shade = has_spheres || H.scene.n_instances > 0 || H.has_delta_lights || H.scene.tri_n != nullptr ||
                                H.scene.tri_uv != nullptr || H.volpath;
        // traversal of one ray queue: the plain kernel, or the two-level one when the scene has instances
        auto trace = [&](TraceArgs &a, bool any_hit, bool classify, cudaStream_t s_) {
#ifndef B200PT_HOST_EMU
            if (tl) {
                a.instances = H.scene.instances;
                a.n_instances = H.scene.n_instances;
                a.tlas_node_off = H.scene.tlas_node_off;
                a.tlas_tri_off = H.scene.tlas_tri_off;
                a.hit_inst_out = a.hit_out == &H.path->hit ? &H.path->hit_inst : nullptr;
                launch_trace2(a, any_hit, classify, r->grid_trace, s_);
                return;
            }
#endif
            launch_trace(a, any_hit, classify, r->instrumented, r->grid_trace, s_);
        };
        auto sphere_args = [&](TraceArgs &a, uint32_t *work) {
            a.sphere_refill_lanes = sphere_refill_lanes();
            a.spheres = H.scene.spheres;
            a.n_spheres = H.scene.n_spheres;
            a.instances = H.scene.instances;
            a.n_instances = tl ? 0u : H.scene.n_instances;
            a.tlas_node_off = H.scene.tlas_node_off;
            a.tlas_tri_off = H.scene.tlas_tri_off;
            a.hit_inst_out = a.hit_out == &H.path->hit ? &H.path->hit_inst : nullptr;
            a.n_tris = (uint32_t)r->scene->n_prims;
            a.sphere_work = work;
        };
        auto trace_path = [&](int b) {
            uint32_t *qc = H.qcount + (size_t)b * Q_PER_BOUNCE;
            uint32_t *wk = H.work + (size_t)b * 16;
            TraceArgs a;
            memset(&a, 0, sizeof(a));
            trace_args_scene(a, r->scene);
            a.materials = H.scene.materials;
            a.stats = H.stats;
            a.stride = REC_F4;
            a.out_stride = (int)sizeof(PathRec);
            a.refill_lanes = r->refill_lanes;
            a.postpone_pct = r->postpone_pct;
            a.ctas = r->trace_ctas;
            a.n_staged = (uint32_t)std::min<uint64_t>((uint64_t)std::max(0, r->stage_nodes), r->scene->n_top_nodes);
            // closest hit of the path rays + classification by BSDF family
            const bool sorted = r->sort_from_bounce >= 0 && b >= r->sort_from_bounce;
            if (sorted) {
                LaunchTimer lt(r, st, 2);
                launch_sort_queue(r->d_dev, H, H.q_path[b & 1], qc + Q_PATH, &H.path->o, &H.path->d, r->grid_shade, st);
            }
            a.ray_o = &H.path->o;
            a.ray_d = &H.path->d;
            a.queue = sorted ? H.q_sorted : H.q_path[b & 1];
            a.count = qc + Q_PATH;
            a.work = wk + 0;
            a.fixed_t_max = INFINITY;
            a.hit_out = &H.path->hit;
            for (int m = 0; m < 4; ++m) a.q_mat[m] = H.q_mat[m];
            a.qcount_mat = qc + Q_MAT0;
            {
                // closest_ms = the traversal launch and, for scenes with spheres, the pass that completes Scene::Intersect;
                // the medium pass below is timed on its own (category 2)
                LaunchTimer lt(r, st, 0);
                // with spheres in the scene the sphere pass decides the final hit, so it does the classification;
                // inside a medium the medium pass does (only paths that reach their surface are shaded)
                trace(a, false, !has_spheres && !medium, st);
                if (has_spheres) {
                    sphere_args(a, wk + 8);
                    launch_spheres(a, false, !medium, r->grid_shade, st);
                    r->launches++;
                }
            }
            if (general) {
                // the medium pass, then -- while some rays reached a medium boundary -- the same two steps again for those
                // rays from behind the boundary (volpath.cpp:115-121: no bounce is spent)
                cudaMemsetAsync(wc, 0, 16 * sizeof(uint32_t), st);
                {
                    LaunchTimer lt2(r, st, 2);
                    launch_medium_general(r->d_dev, H, b, a.queue, qc + Q_PATH, 0, wc + 0, wk + 11, false, r->grid_shade, st);
                }
                for (int cur = 0; device_count(wc + cur, st) != 0; cur ^= 1) {
                    cudaMemsetAsync(wc + (cur ^ 1), 0, sizeof(uint32_t), st);
                    cudaMemsetAsync(wc + 2, 0, 3 * sizeof(uint32_t), st);
                    a.queue = H.q_cross[cur];
                    a.count = wc + cur;
                    a.work = wc + 3;
                    {
                        LaunchTimer lt(r, st, 0);
                        trace(a, false, false, st);
                        sphere_args(a, wc + 4);
                        launch_spheres(a, false, false, r->grid_shade, st);
                        r->launches++;
                    }
                    LaunchTimer lt2(r, st, 2);
                    launch_medium_general(r->d_dev, H, b, H.q_cross[cur], wc + cur, cur ^ 1, wc + (cur ^ 1), wc + 2, true, r->grid_shade, st);
                }
            } else if (medium) {
                LaunchTimer lt2(r, st, 2);
                if (spectral)
                    b200pt_s60::launch_medium(s60(r->d_dev), b, wk + 11, r->grid_shade, st);
                else
                    launch_medium(r->d_dev, b, wk + 11, r->grid_shade, st);
            }
        };
        // Bounded media: the shadow (VisibilityTester::Tr) or MIS (Scene::IntersectTr) rays of bounce b walk from boundary to
        // boundary -- a closest-hit launch per segment, then k_direct_walk ends each ray or sends it on
        auto walk_direct = [&](int b, bool shadow) {
            uint32_t *qc = H.qcount + (size_t)b * Q_PER_BOUNCE;
            uint32_t *wk = H.work + (size_t)b * 16;
            TraceArgs a;
            memset(&a, 0, sizeof(a));
            trace_args_scene(a, r->scene);
            a.materials = H.scene.materials;
            a.stats = H.stats;
            a.stride = REC_F4;
            a.refill_lanes = r->refill_lanes;
            a.postpone_pct = r->postpone_pct;
            a.ctas = r->trace_ctas;
            a.ray_o = shadow ? &H.direct->sh_o : &H.direct->mi_o;
            a.ray_d = shadow ? &H.direct->sh_d : &H.direct->mi_d;
            a.fixed_t_max = shadow ? PT_SHADOW_TMAX : INFINITY;
            a.hit_out = shadow ? H.sh_hit : &H.direct->mis_hit;
            a.out_stride = shadow ? (int)sizeof(uint32_t) : (int)sizeof(DirectRec);
            const uint32_t *queue = shadow ? H.q_shadow : H.q_mis;
            const uint32_t *count = qc + (shadow ? Q_SHADOW : Q_MIS);
            uint32_t *trace_work = wk + (shadow ? 5 : 6), *sphere_work = wk + (shadow ? 9 : 10);
            cudaMemsetAsync(wc, 0, 16 * sizeof(uint32_t), st);
            bool first = true;
            for (int cur = 0;; cur ^= 1) {
                if (!first) {
                    if (device_count(count, st) == 0) break;
                    cudaMemsetAsync(wc + cur, 0, sizeof(uint32_t), st);
                    cudaMemsetAsync(wc + 2, 0, 3 * sizeof(uint32_t), st);
                    trace_work = wc + 3;
                    sphere_work = wc + 4;
                }
                a.queue = queue;
                a.count = count;
                a.work = trace_work;
                {
                    LaunchTimer lt(r, st, 0);
                    trace(a, false, false, st);
                    sphere_args(a, sphere_work);
                    launch_spheres(a, false, false, r->grid_shade, st);
                    r->launches++;
                }
                {
                    LaunchTimer lt2(r, st, 2);
                    launch_direct_walk(r->d_dev, H, shadow, queue, count, cur, wc + cur, wc + 2, !first, r->grid_shade, st);
                }
                queue = H.q_walk[cur];
                count = wc + cur;
                first = false;
            }
        };
        auto trace_direct = [&](int b) {
            if (general) {
                walk_direct(b, true);
                walk_direct(b, false);
                return;
            }
            uint32_t *qc = H.qcount + (size_t)b * Q_PER_BOUNCE;
            uint32_t *wk = H.work + (size_t)b * 16;
            TraceArgs a;
            memset(&a, 0, sizeof(a));
            trace_args_scene(a, r->scene);
            a.materials = H.scene.materials;
            a.stats = H.stats;
            a.stride = REC_F4;
            a.out_stride = (int)sizeof(DirectRec);
            a.refill_lanes = r->refill_lanes;
            a.postpone_pct = r->postpone_pct;
            a.ctas = r->trace_ctas;
            a.n_staged = (uint32_t)std::min<uint64_t>((uint64_t)std::max(0, r->stage_nodes), r->scene->n_top_nodes);
            // shadow rays (any hit), tMax = 1 - ShadowEpsilon
            const bool sorted_sh = r->sort_from_bounce >= 0;
            if (sorted_sh) {
                LaunchTimer lt(r, st2, 2);
                launch_sort_queue(r->d_dev, H, H.q_shadow, qc + Q_SHADOW, &H.direct->sh_o, &H.direct->sh_d, r->grid_shade, st2);
            }
            a.ray_o = &H.direct->sh_o;
            a.ray_d = &H.direct->sh_d;
            a.queue = sorted_sh ? H.q_sorted : H.q_shadow;
            a.count = qc + Q_SHADOW;
            a.work = wk + 5;
            a.fixed_t_max = PT_SHADOW_TMAX;
            a.occ_out = &H.direct->occluded;
            {
                LaunchTimer lt(r, st2, 1);
                trace(a, true, false, st2);
                if (has_spheres) {
                    sphere_args(a, wk + 9);
                    launch_spheres(a, true, false, r->grid_shade, st2);
                    r->launches++;
                }
            }
            // BSDF-sampled MIS rays (closest hit)
            a.ray_o = &H.direct->mi_o;
            a.ray_d = &H.direct->mi_d;
            a.queue = H.q_mis;
            a.count = qc + Q_MIS;
            a.work = wk + 6;
            a.fixed_t_max = INFINITY;
            a.hit_out = &H.direct->mis_hit;
            a.occ_out = nullptr;
            LaunchTimer lt(r, st2, 0);
            trace(a, false, false, st2);
            if (has_spheres) {
                sphere_args(a, wk + 10);
                launch_spheres(a, false, false, r->grid_shade, st2);
                r->launches++;
            }
        };
        trace_path(0);
        for (int b = 0; b <= maxDepth; ++b) {
            uint32_t *wk = H.work + (size_t)b * 16;
            for (int m = 0; m < 4; ++m)
                if (families[m]) {
                    LaunchTimer lt(r, st, 2);
                    if (spectral)
                        b200pt_s60::launch_shade(s60(r->d_dev), m, full_shade, b, wk + 1 + m, r->grid_shade_s60, st);
                    else
                        launch_shade(r->d_dev, m, full_shade, b, wk + 1 + m, r->grid_shade, st);
                }
            if (b < maxDepth && medium) {
                // the medium pass of bounce b+1 writes the same per-slot direct-lighting records: finish bounce b's first
                trace_direct(b);
                {
                    LaunchTimer lt(r, st, 2);
                    if (spectral)
                        b200pt_s60::launch_resolve(s60(r->d_dev), b, wk + 7, r->grid_shade, st);
                    else
                        launch_resolve(r->d_dev, b, wk + 7, r->grid_shade, st);
                }
                trace_path(b + 1);
            } else if (b < maxDepth) {  // no direct lighting is estimated at the last vertex (path.cpp:104)
                if (overlap) {
                    CUDA_TRY(cudaEventRecord(ctx->ev_fork, st));
                    CUDA_TRY(cudaStreamWaitEvent(st2, ctx->ev_fork, 0));
                }
                trace_direct(b);
                if (overlap) CUDA_TRY(cudaEventRecord(ctx->ev_join, st2));
                trace_path(b + 1);
                if (overlap) CUDA_TRY(cudaStreamWaitEvent(st, ctx->ev_join, 0));
                LaunchTimer lt(r, st, 2);
                if (spectral)
                    b200pt_s60::launch_resolve(s60(r->d_dev), b, wk + 7, r->grid_shade, st);
                else
                    launch_resolve(r->d_dev, b, wk + 7, r->grid_shade, st);
            }
        }
        {
            LaunchTimer lt(r, st, 2);
            if (H.filter_general && spectral)
                b200pt_s60::launch_film_general(s60(r->d_dev), s60(H), (uint32_t)first, nb, st);
            else if (H.filter_general)
                launch_film_general(r->d_dev, H, (uint32_t)first, nb, st);
            else if (spectral)
                b200pt_s60::launch_film(s60(r->d_dev), (uint32_t)first, nb, st);
            else
                launch_film(r->d_dev, (uint32_t)first, nb, st);
        }
        launch_accumulate_stats(r->d_dev, 0, st);
        r->launches++;
        CUDA_TRY(cudaGetLastError());
    }
    return B200PT_OK;
}

int b200pt_film_device_buffer(b200pt_render *r, uint64_t *dev_ptr, uint64_t *n_floats) {
    if (!r) return b200pt_fail(B200PT_ERR_INVALID, "render is NULL");
    if (dev_ptr) *dev_ptr = (uint64_t)(uintptr_t)r->host.film;
    if (n_floats) *n_floats = 4ull * (uint64_t)(r->host.crop[2] - r->host.crop[0]) * (r->host.crop[3] - r->host.crop[1]);
    return B200PT_OK;
}

int b200pt_film_read_raw(b200pt_render *r, float *xyzw) {
    if (!r || !xyzw) return b200pt_fail(B200PT_ERR_INVALID, "film_read_raw: NULL argument");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    const size_t n = (size_t)(r->host.crop[2] - r->host.crop[0]) * (r->host.crop[3] - r->host.crop[1]);
    cudaStream_t st = r->scene->ctx->stream;
    CUDA_TRY(cudaMemcpyAsync(xyzw, r->host.film, n * sizeof(float4), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return B200PT_OK;
}

// ---- multi-GPU film merge: NCCL through dlopen (no link-time dependency; the library is usable without it)
namespace {
struct NcclUniqueId {
    char internal[128];
};
struct NcclApi {
    void *lib = nullptr;
    int (*GetUniqueId)(NcclUniqueId *) = nullptr;
    int (*CommInitRank)(void **, int, NcclUniqueId, int) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    int (*Reduce)(const void *, void *, size_t, int, int, int, void *, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    bool ok = false;
};
NcclApi *nccl_api() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return &api;
    tried = true;
    const char *names[] = {getenv("B200PT_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char *nm : names) {
        if (!nm) continue;
        api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
        if (api.lib) break;
    }
    if (!api.lib) return &api;
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(api.lib, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(api.lib, "ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(api.lib, "ncclCommDestroy"));
    api.Reduce = reinterpret_cast<decltype(api.Reduce)>(dlsym(api.lib, "ncclReduce"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(api.lib, "ncclGetErrorString"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.Reduce && api.GetErrorString;
    return &api;
}
}  // namespace

struct b200pt_comm {
    b200pt_ctx *ctx = nullptr;
    void *nccl = nullptr;
    int rank = 0, world = 1;
    bool owned = false;
};

int b200pt_comm_from_nccl(b200pt_ctx *ctx, void *nccl_comm, int rank, int world_size, b200pt_comm **out) {
    if (!ctx || !nccl_comm || !out || world_size < 1 || rank < 0 || rank >= world_size)
        return b200pt_fail(B200PT_ERR_INVALID, "comm_from_nccl: bad argument");
    if (!nccl_api()->ok) return b200pt_fail(B200PT_ERR_INVALID, "comm: libnccl.so.2 could not be loaded (set B200PT_NCCL_LIB)");
    b200pt_comm *c = new b200pt_comm;
    c->ctx = ctx;
    c->nccl = nccl_comm;
    c->rank = rank;
    c->world = world_size;
    *out = c;
    return B200PT_OK;
}

int b200pt_comm_create(b200pt_ctx *ctx, int rank, int world_size, const char *id_file, b200pt_comm **out) {
    if (!ctx || !out || !id_file || world_size < 1 || rank < 0 || rank >= world_size)
        return b200pt_fail(B200PT_ERR_INVALID, "comm_create: bad argument");
    NcclApi *api = nccl_api();
    if (!api->ok) return b200pt_fail(B200PT_ERR_INVALID, "comm_create: libnccl.so.2 could not be loaded (set B200PT_NCCL_LIB)");
    CUDA_TRY(cudaSetDevice(ctx->device));
    NcclUniqueId id;
    memset(&id, 0, sizeof(id));
    if (rank == 0) {
        int rc = api->GetUniqueId(&id);
        if (rc != 0) return b200pt_fail(B200PT_ERR_CUDA, "comm_create: ncclGetUniqueId: %s", api->GetErrorString(rc));
        const std::string tmp = std::string(id_file) + ".tmp";
        FILE *f = fopen(tmp.c_str(), "wb");
        if (!f || fwrite(&id, 1, sizeof(id), f) != sizeof(id)) {
            if (f) fclose(f);
            return b200pt_fail(B200PT_ERR_INVALID, "comm_create: cannot write %s", tmp.c_str());
        }
        fclose(f);
        if (rename(tmp.c_str(), id_file) != 0) return b200pt_fail(B200PT_ERR_INVALID, "comm_create: cannot publish %s", id_file);
    } else {
        bool got = false;
        for (int tries = 0; tries < 2400 && !got; ++tries) {  // up to 120 s
            if (FILE *f = fopen(id_file, "rb")) {
                got = fread(&id, 1, sizeof(id), f) == sizeof(id);
                fclose(f);
            }
            if (!got) std::this_thread::sleep_for(std::chrono::milliseconds(50));
        }
        if (!got) return b200pt_fail(B200PT_ERR_INVALID, "comm_create: rank %d never saw the NCCL id in %s", rank, id_file);
    }
    void *comm = nullptr;
    int rc = api->CommInitRank(&comm, world_size, id, rank);
    if (rc != 0) return b200pt_fail(B200PT_ERR_CUDA, "comm_create: ncclCommInitRank: %s", api->GetErrorString(rc));
    b200pt_comm *c = new b200pt_comm;
    c->ctx = ctx;
    c->nccl = comm;
    c->rank = rank;
    c->world = world_size;
    c->owned = true;
    *out = c;
    return B200PT_OK;
}

void b200pt_comm_destroy(b200pt_comm *c) {
    if (!c) return;
    if (c->owned && c->nccl && nccl_api()->ok) {
        cudaSetDevice(c->ctx->device);
        nccl_api()->CommDestroy(c->nccl);
    }
    delete c;
}

int b200pt_film_reduce(b200pt_render *r, b200pt_comm *c, int root) {
    if (!r || !c) return b200pt_fail(B200PT_ERR_INVALID, "film_reduce: NULL argument");
    if (root < 0 || root >= c->world) return b200pt_fail(B200PT_ERR_INVALID, "film_reduce: root %d out of range", root);
    if (c->ctx != r->scene->ctx) return b200pt_fail(B200PT_ERR_INVALID, "film_reduce: communicator and render belong to different contexts");
    CUDA_TRY(cudaSetDevice(c->ctx->device));
    const size_t n = 4 * (size_t)(r->host.crop[2] - r->host.crop[0]) * (r->host.crop[3] - r->host.crop[1]);
    // ncclFloat = 7, ncclSum = 0 (nccl.h); in place: send == recv
    const int rc = nccl_api()->Reduce(r->host.film, r->host.film, n, 7, 0, root, c->nccl, c->ctx->stream);
    if (rc != 0) return b200pt_fail(B200PT_ERR_CUDA, "film_reduce: ncclReduce: %s", nccl_api()->GetErrorString(rc));
    return B200PT_OK;
}

int b200pt_film_read_rgb(b200pt_render *r, float *rgb_out) {
    if (!r || !rgb_out) return b200pt_fail(B200PT_ERR_INVALID, "film_read_rgb: NULL argument");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    const size_t n = (size_t)(r->host.crop[2] - r->host.crop[0]) * (r->host.crop[3] - r->host.crop[1]);
    cudaStream_t st = r->scene->ctx->stream;
    if (!r->d_rgb) {  // staging buffer of the WriteImage pipeline, kept for the lifetime of the render object
        cudaError_t ea = dev_alloc(r, &r->d_rgb, n * 3);
        if (ea != cudaSuccess) return b200pt_fail(B200PT_ERR_OOM, "film_read_rgb: cudaMalloc failed: %s", cudaGetErrorString(ea));
    }
    launch_film_rgb(r->host.film, r->d_rgb, (int)n, r->film.scale, st);
    cudaError_t e = cudaMemcpyAsync(rgb_out, r->d_rgb, n * 3 * sizeof(float), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return b200pt_fail(B200PT_ERR_CUDA, "film_read_rgb: %s", cudaGetErrorString(e));
    return B200PT_OK;
}

int b200pt_debug_sobol(b200pt_render *r, int32_t px, int32_t py, int64_t sample, int32_t dim0, int32_t n, float *out) {
    if (!r || !out || n <= 0 || dim0 < 0 || dim0 + n > r->host.sampler.n_dims)
        return b200pt_fail(B200PT_ERR_INVALID, "debug_sobol: bad argument");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    cudaStream_t st = r->scene->ctx->stream;
    float *d = nullptr;
    CUDA_TRY(cudaMalloc(&d, n * sizeof(float)));
    launch_debug_sobol(r->d_dev, px, py, sample, dim0, n, d, st);
    cudaError_t e = cudaMemcpyAsync(out, d, n * sizeof(float), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    if (e != cudaSuccess) return b200pt_fail(B200PT_ERR_CUDA, "debug_sobol: %s", cudaGetErrorString(e));
    return B200PT_OK;
}

int b200pt_debug_camera_rays(b200pt_render *r, int32_t px, int32_t py, int32_t n, b200pt_ray *out) {
    if (!r || !out || n <= 0) return b200pt_fail(B200PT_ERR_INVALID, "debug_camera_rays: bad argument");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    cudaStream_t st = r->scene->ctx->stream;
    b200pt_ray *d = nullptr;
    CUDA_TRY(cudaMalloc(&d, n * sizeof(b200pt_ray)));
    launch_debug_camera(r->d_dev, px, py, n, d, st);
    cudaError_t e = cudaMemcpyAsync(out, d, n * sizeof(b200pt_ray), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    if (e != cudaSuccess) return b200pt_fail(B200PT_ERR_CUDA, "debug_camera_rays: %s", cudaGetErrorString(e));
    return B200PT_OK;
}

// Renders the pixel's tile into the per-slot radiance buffer and returns the
// guarded per-sample values (film accumulation is undone by saving/restoring the film).
int b200pt_debug_pixel_samples(b200pt_render *r, int32_t px, int32_t py, float *out_rgb) {
    if (!r || !out_rgb) return b200pt_fail(B200PT_ERR_INVALID, "debug_pixel_samples: NULL argument");
    const RenderDev &H = r->host;
    if (px < H.sampler.sb[0] || px >= H.sampler.sb[2] || py < H.sampler.sb[1] || py >= H.sampler.sb[3])
        return b200pt_fail(B200PT_ERR_INVALID, "debug_pixel_samples: pixel outside the sample bounds");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    cudaStream_t st = r->scene->ctx->stream;
    const size_t npx = (size_t)(H.crop[2] - H.crop[0]) * (H.crop[3] - H.crop[1]);
    float4 *saved = nullptr;
    CUDA_TRY(cudaMalloc(&saved, npx * sizeof(float4)));
    CUDA_TRY(cudaMemcpyAsync(saved, H.film, npx * sizeof(float4), cudaMemcpyDeviceToDevice, st));
    const int tx = (px - H.sampler.sb[0]) / 16, ty = (py - H.sampler.sb[1]) / 16;
    int32_t tile = ty * H.tiles_x + tx;
    int rc = b200pt_render_tiles(r, &tile, 1);
    if (rc == B200PT_OK) {
        const uint32_t pix = (uint32_t)((py - (H.sampler.sb[1] + ty * 16)) * 16 + (px - (H.sampler.sb[0] + tx * 16)));
        const int ns = r->scene->nspec;
        std::vector<PathRec> tmp((size_t)r->spp);
        std::vector<float> bins((size_t)r->spp * (size_t)std::max(ns, 1));
        cudaError_t e = cudaMemcpyAsync(tmp.data(), H.path + (size_t)pix * r->spp, (size_t)r->spp * sizeof(PathRec),
                                        cudaMemcpyDeviceToHost, st);
        if (ns && e == cudaSuccess)  // slot-major [capacity][bins]: the pixel's samples are consecutive slots
            e = cudaMemcpyAsync(bins.data(), H.s_L + (size_t)pix * r->spp * ns, (size_t)r->spp * ns * sizeof(float),
                                cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(H.film, saved, npx * sizeof(float4), cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) rc = b200pt_fail(B200PT_ERR_CUDA, "debug_pixel_samples: %s", cudaGetErrorString(e));
        for (int i = 0; i < r->spp && rc == B200PT_OK; ++i) {
            if (!ns) {
                Spec L = rgb(tmp[i].L.x, tmp[i].L.y, tmp[i].L.z);
                if (has_nans(L) || lum(L) < -1e-5f || pt_isinf(lum(L))) L = rgb1(0.f);  // integrator.cpp:294-315
                out_rgb[3 * i] = L.c[0];
                out_rgb[3 * i + 1] = L.c[1];
                out_rgb[3 * i + 2] = L.c[2];
                continue;
            }
            // SampledSpectrum host: the sample as ToXYZ -> XYZToRGB reports it (spectrum.h:380-392, :56-60)
            std::vector<float> L((size_t)ns);
            bool nan = false;
            for (int b = 0; b < ns; ++b) {
                L[b] = bins[(size_t)i * ns + b];
                nan = nan || pt_isnan(L[b]);
            }
            const float y = host_spectrum_y(r->scene, L);
            if (nan || y < -1e-5f || pt_isinf(y)) std::fill(L.begin(), L.end(), 0.f);
            const float *cie = r->scene->cie_xyz.data();
            float xyz[3] = {0.f, 0.f, 0.f};
            for (int b = 0; b < ns; ++b) {
                xyz[0] += cie[b] * L[b];
                xyz[1] += cie[ns + b] * L[b];
                xyz[2] += cie[2 * ns + b] * L[b];
            }
            const float scale = float(700 - 400) / float(106.856895f * ns);
            for (int k = 0; k < 3; ++k) xyz[k] *= scale;
            xyz_to_rgb(xyz, out_rgb + 3 * i);
        }
    }
    cudaFree(saved);
    return rc;
}

int b200pt_get_stats(b200pt_render *r, b200pt_stats *out) {
    if (!r || !out) return b200pt_fail(B200PT_ERR_INVALID, "get_stats: NULL argument");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    cudaStream_t st = r->scene->ctx->stream;
    unsigned long long h[9];
    CUDA_TRY(cudaMemcpyAsync(h, r->host.stats, sizeof(h), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    drain_timers(r);
    memset(out, 0, sizeof(*out));
    out->camera_rays = h[0];
    out->regular_rays = h[1];
    out->shadow_rays = h[2];
    out->nodes_visited = h[3];
    out->tris_tested = h[4];
    out->any_nodes_visited = h[5];
    out->any_tris_tested = h[6];
    out->closest_launches = r->launches_cat[0];
    out->any_launches = r->launches_cat[1];
    out->closest_ms = r->ms[0];
    out->any_ms = r->ms[1];
    out->shade_ms = r->ms[2];
    out->launches = r->launches;
    out->stack_overflows = h[7];
    out->dimension_overflows = h[8];
    return B200PT_OK;
}

int b200pt_reset_stats(b200pt_render *r) {
    if (!r) return b200pt_fail(B200PT_ERR_INVALID, "render is NULL");
    CUDA_TRY(cudaSetDevice(r->scene->ctx->device));
    cudaStream_t st = r->scene->ctx->stream;
    CUDA_TRY(cudaStreamSynchronize(st));
    drain_timers(r);
    CUDA_TRY(cudaMemsetAsync(r->host.stats, 0, 9 * sizeof(unsigned long long), st));
    r->ms[0] = r->ms[1] = r->ms[2] = 0;
    r->launches = 0;
    r->launches_cat[0] = r->launches_cat[1] = r->launches_cat[2] = 0;
    return B200PT_OK;
}

int b200pt_render_set_option(b200pt_render *r, const char *name, int value) {
    if (!r || !name) return b200pt_fail(B200PT_ERR_INVALID, "set_option: NULL argument");
    if (!strcmp(name, "instrument"))
        r->instrumented = value != 0;
    else if (!strcmp(name, "profile"))
        r->profiling = value != 0;
    else if (!strcmp(name, "refill_lanes"))
        r->refill_lanes = value;
    else if (!strcmp(name, "postpone_pct"))
        r->postpone_pct = value;
    else if (!strcmp(name, "trace_ctas"))
        r->trace_ctas = value;
    else if (!strcmp(name, "stage_nodes"))
        r->stage_nodes = value < 0 ? 0 : (value > 512 ? 512 : value);
    else if (!strcmp(name, "overlap"))
        r->overlap = value != 0;
    else
        return b200pt_fail(B200PT_ERR_INVALID, "set_option: unknown option %s", name);
    return B200PT_OK;
}

}  // extern "C"
