/* b200pt.h -- C ABI of the H100-native path-tracing hot path.
 *
 * This is the drop-in boundary for ONE path of pbrt-v3(-distributed): the
 * per-tile SamplerIntegrator::Render loop (core/integrator.cpp:228-339) with
 * PathIntegrator::Li (integrators/path.cpp:64-188), BVHAccel::Intersect /
 * IntersectP (accelerators/bvh.cpp:662-738), Triangle::Intersect
 * (shapes/triangle.cpp:188-425), the Sobol' sampler (samplers/sobol.cpp:42-59),
 * the perspective camera (cameras/perspective.cpp:95-144), the four materials
 * matte/plastic/metal/glass, diffuse area lights with MIS direct lighting
 * (core/integrator.cpp:85-215) and the box-filtered film
 * (core/film.h:121-161, core/film.cpp:117-130).  Widened since (each descriptor
 * says where): the Halton sampler, Sphere shapes and sphere lights, object
 * instances, the mirror material, point / spot / distant lights, every pixel
 * filter, SampledSpectrum hosts (60-bin spectra), VolPathIntegrator
 * (integrators/volpath.cpp:60-188) with one homogeneous medium around the scene,
 * infinite area lights, and image textures (textures/imagemap.h) on RGB hosts.
 *
 * The reference has no FFI: its "plugins" are C++ subclasses picked by name in
 * RenderOptions::MakeIntegrator (core/api.cpp:1666-1718).  A host integrator
 * (pbrt-v3-distributed_b200/host/gpupath.cpp, GpuIntegrator<PathIntegrator> and
 * GpuIntegrator<VolPathIntegrator>, Integrator::Render integrator.h:53-58) flattens the parsed Scene into the
 * plain-old-data descriptors below and calls these entry points; see
 * INTEGRATION.md for the binding.  Everything is `extern "C"`, plain pointers
 * and sizes; no torch / CUDA types appear in any signature (device pointers
 * travel as uint64_t).
 *
 * Conventions: every function returns 0 on success and a negative
 * b200pt_status on failure; b200pt_last_error() gives the message (thread
 * local).  The caller owns all host arrays passed to b200pt_scene_create for
 * the duration of the call; the library copies what it needs to the device and
 * owns all device memory behind a handle.  There is NO CPU fallback: if no
 * CUDA device is usable every compute entry point fails with
 * B200PT_ERR_NO_DEVICE.
 */
#ifndef B200PT_H
#define B200PT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200PT_ABI_VERSION 6
#define B200PT_SPECTRUM_SAMPLES 60  /* nSpectralSamples, core/spectrum.h:52 */
#define B200PT_MATERIAL_SPECTRA 5

typedef enum b200pt_status {
    B200PT_OK = 0,
    B200PT_ERR_INVALID = -1,     /* bad argument / unsupported feature        */
    B200PT_ERR_NO_DEVICE = -2,   /* no usable CUDA device (no CPU fallback)   */
    B200PT_ERR_CUDA = -3,        /* a CUDA runtime call failed                */
    B200PT_ERR_OOM = -4          /* device or host allocation failed          */
} b200pt_status;

/* ---- materials: materials/{matte,plastic,metal,glass}.cpp ---------------- */
typedef enum b200pt_material_type {
    B200PT_MAT_MATTE = 0,   /* LambertianReflection(Kd) or, variant 1, OrenNayar(Kd, sigma)   matte.cpp:45-62 */
    B200PT_MAT_PLASTIC = 1, /* Lambertian(Kd)+MicrofacetReflection(Ks,TR(a,a),FrDielectric(1.5,1)) plastic.cpp:45-70 */
    B200PT_MAT_METAL = 2,   /* MicrofacetReflection(1,TR(ax,ay),FrConductor(1,eta,k))   metal.cpp:59-80 */
    B200PT_MAT_GLASS = 3,   /* FresnelSpecular(R,T,1,index) (smooth, glass.cpp:62-64) or, variant 1, rough glass:
                               MicrofacetReflection(R,TR,FrDielectric(1,index)) + MicrofacetTransmission(T,TR,1,index)
                               glass.cpp:65-90; variant 2 is MirrorMaterial (materials/mirror.cpp:45-56), which shares the
                               specular family: SpecularReflection(ks, FresnelNoOp), BSDF eta 1 */
    B200PT_MAT_NONE = 4     /* null material: GetMaterial()==nullptr is NOT supported; reserved */
} b200pt_material_type;

/* Constant textures (textures/constant.h) are evaluated by the host, which also
 * applies TrowbridgeReitzDistribution::RoughnessToAlpha (microfacet.h:123-128)
 * itself, so alpha_x/alpha_y below are the final alphas. Spectra are RGB
 * (core/spectrum.h:429), already Clamp()ed like the materials do.  On RGBSpectrum
 * hosts a parameter may instead be an ImageTexture under UVMapping2D
 * (b200pt_scene_bind_texture): the device then evaluates it per hit, clamps and
 * remaps it like the material does, and the value here is ignored. */
typedef struct b200pt_material {
    int32_t type;        /* b200pt_material_type */
    float kd[3];         /* matte Kd, plastic Kd                      */
    float ks[3];         /* plastic Ks, glass Kr (R)                  */
    float kt[3];         /* glass Kt (T)                              */
    float eta[3];        /* metal eta (RGB)                           */
    float k[3];          /* metal k   (RGB)                           */
    float alpha_x;       /* TR alpha (plastic: ax==ay); matte variant 1: OrenNayar A (reflection.h:416-419) */
    float alpha_y;       /*                               matte variant 1: OrenNayar B                      */
    float index;         /* glass index of refraction (BSDF::eta)     */
    int32_t variant;     /* 0 = default lobe set, 1 / 2 = see the material types above */
} b200pt_material;

/* ---- lights.  Order == Scene::lights order (it decides lightNum).  kind 0: one
 * DiffuseAreaLight per emissive triangle or sphere (api.cpp:1357-1364,
 * lights/diffuse.cpp:42-87).  kinds 1-3: the delta lights PointLight
 * (lights/point.cpp:43-56), SpotLight (lights/spot.cpp:42-76) and DistantLight
 * (lights/distant.cpp:43-66): no geometry, no BSDF-sampling branch in
 * EstimateDirect (integrator.cpp:166). */
enum { B200PT_LIGHT_AREA = 0, B200PT_LIGHT_POINT = 1, B200PT_LIGHT_SPOT = 2, B200PT_LIGHT_DISTANT = 3,
       /* InfiniteAreaLight (lights/infinite.cpp:43-132), PathIntegrator on RGBSpectrum hosts only: world_to_light and
        * world_radius (0 = computed from the scene bounds) are used here, the map and its sampling tables are set with
        * b200pt_scene_set_infinite_light before b200pt_render_create */
       B200PT_LIGHT_INFINITE = 4 };
typedef struct b200pt_area_light {
    int32_t triangle;    /* area light: index into the triangle arrays                */
    float lemit[3];      /* area: Lemit; point / spot: I; distant: L (all already multiplied by "scale") */
    int32_t two_sided;   /* area: "twosided" parameter                                */
    int32_t sphere;      /* area: -1, or index into spheres[]: the light's shape is that sphere and
                            `triangle` is ignored                                      */
    int32_t kind;        /* B200PT_LIGHT_*                                             */
    float position[3];   /* point / spot: pLight; distant: wLight (normalised, towards the light) */
    float cos_total_width, cos_falloff_start;  /* spot (spot.cpp:50-51)                */
    float world_to_light[16];                  /* spot: Light::WorldToLight.m           */
    float world_radius;  /* distant: DistantLight::worldRadius (distant.h:54-58); 0 = computed from the scene bounds */
} b200pt_area_light;

/* ---- spheres: Sphere shapes (shapes/sphere.cpp:49-306), full or clipped by
 * zmin / zmax / phimax.  A sphere keeps
 * its object space like in the reference: both matrices are the host's own
 * Transform::m / mInv (row-major).  Spheres are tested outside the triangle
 * BVH (there are few of them: lights, a handful of objects). */
typedef struct b200pt_sphere {
    float object_to_world[16];          /* Shape::ObjectToWorld->m                      */
    float world_to_object[16];          /* Shape::WorldToObject->m (== ObjectToWorld->mInv) */
    float radius;
    int32_t material_id;                /* index into materials                          */
    int32_t light_id;                   /* index into lights or -1                       */
    uint8_t reverse_orientation;        /* Shape::reverseOrientation                     */
    uint8_t transform_swaps_handedness; /* Shape::transformSwapsHandedness               */
    uint8_t pad[2];
    /* Bounds (min xyz, max xyz) of the accelerator leaf that holds the sphere in the host's BVHAccel.  The
     * reference only calls Sphere::Intersect(P) on rays that pass Bounds3::IntersectP on that leaf with the
     * current ray.tMax (accelerators/bvh.cpp:676,713, core/geometry.h:1411-1438), and Sphere::Intersect's own
     * root can be off by more than the box test's error, so the box test decides real cases (a shadow ray
     * towards the limb of a distant sphere light).  All zeros = use the sphere's own Shape::WorldBound(). */
    float leaf_bounds[6];
    /* The Sphere's own members (sphere.h:55-61, :66-68) for a partial sphere: zMin, zMax (already clamped and
     * ordered), thetaMin, thetaMax, phiMax (radians).  phi_max == 0 means a full sphere and the five values are
     * ignored (-r, r, acos(-1), acos(1), Radians(360) are used).  b200pt_host_sphere_params computes them from the
     * shape's parameters for hosts that do not have a Sphere object. */
    float z_min, z_max, theta_min, theta_max, phi_max;
} b200pt_sphere;

/* ---- object instances: TransformedPrimitive (core/primitive.cpp:70-98) over
 * the triangles of an "ObjectBegin" block (api.cpp:1500-1592).  The object's
 * triangles are a contiguous range of the scene's triangle arrays *behind* the
 * n_toplevel_triangles ordinary ones, in the object's own space (what the
 * reference keeps in its TriangleMesh); instances of the same object name the
 * same range.  Rays are transformed into the object (Transform::operator()(Ray),
 * transform.h:251-264), intersected there, and the hit is transformed back
 * (transform.cpp:262-297) like the reference does.  Area lights cannot sit
 * inside instances (api.cpp:1411-1413); animated instance transforms are out
 * of scope. */
typedef struct b200pt_instance {
    int64_t first_triangle;        /* range of the object's triangles                       */
    int64_t n_triangles;
    float instance_to_world[16];   /* TransformedPrimitive::PrimitiveToWorld.startTransform->m */
    float world_to_instance[16];   /* ... ->mInv                                             */
    int32_t is_identity;           /* Transform::IsIdentity(): the hit is not transformed back (primitive.cpp:93-94) */
    float leaf_bounds[6];          /* bounds of the top-level BVH leaf holding the instance (see b200pt_sphere);
                                      all zeros = the instance's own WorldBound()            */
    int32_t pad;
} b200pt_instance;

/* ---- scene: world-space triangle soup + per-triangle attributes ---------
 * Triangle i is the i-th GeometricPrimitive handed to the accelerator
 * (accelerators/bvh.cpp:183).  Vertices are the world-space TriangleMesh::p
 * values (shapes/triangle.cpp:73-75) gathered through the index buffer:
 * 9 floats per triangle (p0 p1 p2).  Per-vertex shading normals (TriangleMesh::n,
 * world space) and uvs (TriangleMesh::uv) are optional, gathered the same way;
 * per-vertex tangents (s) are out of scope and must be rejected by the host.
 * Alpha masks are set after creation (b200pt_scene_set_alpha_masks). */
typedef struct b200pt_scene_desc {
    int64_t n_triangles;
    const float *vertices;        /* [n_triangles][3][3]                              */
    const int32_t *material_id;   /* [n_triangles] index into materials               */
    const int32_t *light_id;      /* [n_triangles] index into lights or -1            */
    const uint8_t *flip_normal;   /* [n_triangles] reverseOrientation ^ transformSwapsHandedness
                                     (shapes/triangle.cpp:420-421); may be NULL (=0)  */
    int32_t n_materials;
    const b200pt_material *materials;
    int32_t n_lights;
    const b200pt_area_light *lights;
    /* optional per-vertex shading data (shapes/triangle.cpp:293-425); NULL = none */
    const float *normals;         /* [n_triangles][3][3] world-space n of the three vertices  */
    const float *uvs;             /* [n_triangles][3][2]                                      */
    const uint8_t *vertex_flags;  /* [n_triangles] bit0: triangle's mesh has normals, bit1: has uvs;
                                     NULL = every triangle has whatever arrays are non-NULL   */
    int32_t n_spheres;
    const b200pt_sphere *spheres; /* [n_spheres]                                              */
    /* object instancing: triangles [n_toplevel_triangles, n_triangles) belong to objects (see b200pt_instance);
     * with n_instances == 0 every triangle is a top-level one and n_toplevel_triangles is ignored */
    int32_t n_instances;
    const b200pt_instance *instances;
    int64_t n_toplevel_triangles;
    /* Hosts built with `typedef SampledSpectrum Spectrum` (core/pbrt.h:124-125, core/spectrum.h:283-427) pass their
     * spectra as they hold them: B200PT_SPECTRUM_SAMPLES bins each, and SampledSpectrum::X/Y/Z (spectrum.cpp:80-100)
     * for y() and ToXYZ().  The RGB triples of materials and lights are then ignored.  0 = RGBSpectrum host. */
    int32_t n_spectrum_samples;     /* 0 or B200PT_SPECTRUM_SAMPLES                                        */
    int32_t reserved_spectral;
    const float *material_spectra;  /* [n_materials][B200PT_MATERIAL_SPECTRA][60]: kd, ks, kt, eta, k        */
    const float *light_spectra;     /* [n_lights][60]: Lemit / I / L, multiplied by "scale" like lemit      */
    const float *cie_xyz;           /* [3][60]: SampledSpectrum::X, Y, Z                                    */
} b200pt_scene_desc;

/* ---- camera: PerspectiveCamera (cameras/perspective.cpp:45-144) ----------
 * The two matrices are the host's own Transform::m values (row-major,
 * core/transform.h:60-80): RasterToCamera (camera.h:104) and the static
 * CameraToWorld.  Animated cameras are out of scope. */
typedef struct b200pt_camera_desc {
    float raster_to_camera[16];
    float camera_to_world[16];
    float lens_radius;       /* > 0 enables the thin lens branch :104-116 */
    float focal_distance;
    float shutter_open;
    float shutter_close;
} b200pt_camera_desc;

/* ---- film: Film + pixel filter (core/film.cpp:44-130, core/film.h:121-161) --
 * The filter is what Film keeps of it: its radius and the 16x16 table of
 * weights Film's constructor evaluates (film.cpp:68-77) -- the host passes its
 * own table, so every Filter subclass works and no filter function is
 * evaluated here.  filter_table == NULL means the default BoxFilter (all
 * weights 1, box.cpp:41-43), for which radius 0.5 takes a specialised path. */
typedef struct b200pt_film_desc {
    int32_t full_resolution[2];
    int32_t cropped_bounds[4];     /* croppedPixelBounds x0 y0 x1 y1 (film.cpp:54-58) */
    float filter_radius[2];        /* Filter::radius (<= 8 pixels)                    */
    float scale;                   /* Film::scale                                     */
    float max_sample_luminance;    /* Film::maxSampleLuminance (INFINITY = off)       */
    const float *filter_table;     /* [16][16] Film::filterTable, or NULL             */
} b200pt_film_desc;

/* ---- sampler: SobolSampler (samplers/sobol.h:45-69) or HaltonSampler
 * (samplers/halton.h:48-83), both GlobalSamplers (core/sampler.cpp:136-195).
 * The tables stay the host's data.  Sobol': the host passes SobolMatrices32 and
 * the two rows VdCSobolMatrices[log2res-1], VdCSobolMatricesInv[log2res-1] it
 * already owns (core/sobolmatrices.cpp).  Halton: the host passes
 * HaltonSampler::radicalInversePermutations (halton.cpp:69-72, built by
 * ComputeRadicalInversePermutations, lowdiscrepancy.cpp:2490-2504): the digit
 * permutation of base Primes[d] starts at PrimeSums[d]; only the first
 * n_dimensions bases are read.  baseScales / baseExponents / sampleStride /
 * multInverse (halton.cpp:74-92) are recomputed by the library from
 * sample_bounds. */
enum { B200PT_SAMPLER_SOBOL = 0, B200PT_SAMPLER_HALTON = 1 };
typedef struct b200pt_sampler_desc {
    int32_t samples_per_pixel;     /* Sobol': already rounded up to a power of two (sobol.h:52) */
    int32_t sample_bounds[4];      /* Film::GetSampleBounds() x0 y0 x1 y1             */
    int32_t n_dimensions;          /* Sobol': rows in matrices32 (<=1024); Halton: bases covered (<=1000) */
    const uint32_t *matrices32;    /* [n_dimensions][52]  SobolMatrices32             */
    const uint64_t *vdc;           /* [52] VdCSobolMatrices[log2Resolution-1]         */
    const uint64_t *vdc_inv;       /* [52] VdCSobolMatricesInv[log2Resolution-1]      */
    int32_t type;                  /* B200PT_SAMPLER_*                                */
    int32_t reserved;
    const uint16_t *halton_permutations; /* [PrimeSums[n_dimensions]] (Halton only)   */
} b200pt_sampler_desc;

/* ---- integrator: PathIntegrator parameters (integrators/path.cpp:190-213) */
typedef enum b200pt_light_strategy {
    B200PT_LIGHTS_UNIFORM = 0,     /* UniformLightDistribution  lightdistrib.cpp:68-75 */
    B200PT_LIGHTS_POWER = 1,       /* PowerLightDistribution    lightdistrib.cpp:77-82 */
    B200PT_LIGHTS_SPATIAL = 2      /* SpatialLightDistribution  lightdistrib.cpp:96-300 (pbrt's default): every
                                      voxel's distribution is a pure function of the voxel, so all of them are
                                      computed up front on the device instead of lazily */
} b200pt_light_strategy;

typedef struct b200pt_medium {     /* HomogeneousMedium(sigma_a, sigma_s, g), homogeneous.h:50-54 */
    int32_t present;
    float sigma_a[3];              /* already multiplied by "scale" (api.cpp:697-700) */
    float sigma_s[3];
    float g;                       /* Henyey-Greenstein asymmetry (core/medium.h:69-72) */
    const float *spectra;          /* SampledSpectrum hosts (scene n_spectrum_samples == 60): [2][60] = sigma_a, sigma_s
                                      as the host holds them; the RGB triples are then ignored.  NULL otherwise */
} b200pt_medium;

typedef struct b200pt_integrator_desc {
    int32_t max_depth;             /* "maxdepth", default 5          */
    float rr_threshold;            /* "rrthreshold", default 1       */
    int32_t light_strategy;        /* b200pt_light_strategy          */
    int32_t pixel_bounds[4];       /* "pixelbounds" ∩ sample bounds, x0 y0 x1 y1 (path.cpp:195-207) */
    /* VolPathIntegrator (integrators/volpath.cpp:60-188) instead of PathIntegrator: a light is sampled at every vertex
     * (also purely specular ones, :124-128) and, with `medium.present`, every ray travels through one
     * HomogeneousMedium (media/homogeneous.cpp) that surrounds the whole scene -- the camera is in it and no surface is
     * a medium transition.  Heterogeneous media are not supported. */
    int32_t volumetric;
    b200pt_medium medium;
    /* Media bounded by surfaces (ABI 6): Sphere shapes with `Material ""` under `MediumInterface "inside" "outside"`
     * (api.cpp:1032-1045, primitive.cpp:106-127).  sphere_medium[k] >= 0 makes sphere k of the scene such a boundary:
     * no BSDF (the path steps over it without spending a bounce, volpath.cpp:115-121), inside it is
     * bounded_media[sphere_medium[k]], outside it the medium above (or vacuum); a ray's medium switches by the side it
     * leaves on (interaction.h:80-82), shadow and MIS rays accumulate transmittance segment by segment
     * (light.cpp:63-81, scene.cpp:57-70).  Such a sphere must not be a light.  n_bounded_media == 0: none. */
    int32_t n_bounded_media;
    int32_t reserved;
    const b200pt_medium *bounded_media;  /* [n_bounded_media]; `present` is ignored */
    const int32_t *sphere_medium;        /* [scene n_spheres]: index into bounded_media, or -1 for an ordinary sphere */
} b200pt_integrator_desc;

/* ---- per-ray records for the kernel-level entry points ------------------ */
typedef struct b200pt_ray {
    float o[3];
    float t_max;
    float d[3];
    float pad;
} b200pt_ray;                      /* 32 B */

typedef struct b200pt_hit {
    int32_t triangle;              /* -1 = miss                                       */
    float t;                       /* Triangle::Intersect tHit                        */
    float b0, b1;                  /* barycentrics (b2 recomputed as in :268)         */
} b200pt_hit;                      /* 16 B */

/* ---- counters mirroring the reference's STAT_COUNTERs ------------------- */
typedef struct b200pt_stats {
    uint64_t camera_rays;          /* "Integrator/Camera rays traced"   integrator.cpp:48  */
    uint64_t regular_rays;         /* "Intersections/Regular ray intersection tests" scene.cpp:40 */
    uint64_t shadow_rays;          /* "Intersections/Shadow ray intersection tests"  scene.cpp:41 */
    uint64_t nodes_visited;        /* wide-BVH nodes fetched by closest-hit launches ("instrument") */
    uint64_t tris_tested;          /* ray-triangle tests in closest-hit launches                    */
    uint64_t any_nodes_visited;    /* same for the any-hit (shadow) launches                        */
    uint64_t any_tris_tested;
    double closest_ms;             /* device time in closest-hit traversal launches   */
    double any_ms;                 /* device time in any-hit traversal launches       */
    double shade_ms;               /* device time in all other launches               */
    uint64_t launches;             /* kernels launched by the library                 */
    uint64_t closest_launches;     /* of which closest-hit traversal                  */
    uint64_t any_launches;         /* of which any-hit traversal                      */
    uint64_t stack_overflows;      /* child groups a full traversal stack had to drop (must be 0: a non-zero
                                      count means hits may have been missed; scene_create rejects trees whose
                                      depth could overflow, so this is a tripwire, not an expected event)   */
    uint64_t dimension_overflows;  /* paths ended because their sampler dimension ran past n_dimensions (only
                                      possible with bounded media: every boundary crossed inside a medium spends
                                      two dimensions without spending a bounce; the reference aborts there)    */
} b200pt_stats;

typedef struct b200pt_ctx b200pt_ctx;      /* device + stream                          */
typedef struct b200pt_scene b200pt_scene;  /* device-resident triangles + wide BVH     */
typedef struct b200pt_render b200pt_render;/* camera+film+sampler+integrator + film buffers */

/* ---- library ------------------------------------------------------------ */
int b200pt_abi_version(void);
const char *b200pt_last_error(void);

/* Binds to CUDA device `device` (cudaSetDevice) and creates the stream all
 * work of this context runs on. */
int b200pt_ctx_create(int device, b200pt_ctx **out);
void b200pt_ctx_destroy(b200pt_ctx *ctx);
int b200pt_ctx_synchronize(b200pt_ctx *ctx);
/* cudaStream_t of the context as an integer (for CUDA-event timing by the caller). */
uint64_t b200pt_ctx_stream(b200pt_ctx *ctx);
/* Context options.  "gpu_bvh_build" (0/1, default 0; the environment variable B200PT_BVH_BUILD=gpu|host overrides
 * it): build the acceleration structure on the device (Morton order -> binary radix tree -> 8-wide collapse) instead
 * of the host SAH builder.  Both replace BVHAccel's constructor (accelerators/bvh.cpp:183-225); results are
 * identical (hits are decided by the exact triangle test), the device build is faster to build and slightly slower
 * to traverse on some scenes. */
int b200pt_ctx_set_option(b200pt_ctx *ctx, const char *key, int64_t value);

/* ---- scene: replaces CreateBVHAccelerator (accelerators/bvh.cpp:740-760) --
 * Builds the 8-wide compressed BVH on the host (SAH) and uploads it. */
int b200pt_scene_create(b200pt_ctx *ctx, const b200pt_scene_desc *desc, b200pt_scene **out);
void b200pt_scene_destroy(b200pt_scene *scene);
/* Re-uploads the scene's nodes, triangle records and materials from the
 * library's pinned host copies (asynchronous on the context's stream).  This is
 * the host->device traffic of one end-to-end render; returns the bytes copied. */
int b200pt_scene_upload(b200pt_scene *scene, uint64_t *bytes);
/* bytes of device memory held by nodes / triangles, node count */
int b200pt_scene_info(const b200pt_scene *scene, uint64_t *node_bytes, uint64_t *tri_bytes,
                      uint64_t *n_nodes);

/* ---- infinite area lights: what InfiniteAreaLight (lights/infinite.cpp:43-84) holds, copied, never recomputed.
 * Le and Sample_Li look the map up with width 0, which is the bilinear lookup of pyramid level 0 with Repeat wrap
 * (MIPMap::Lookup / triangle, mipmap.h:245-273): level 0 is all the device needs.  The Distribution2D
 * (sampling.h:124-141) is passed as the host built it from the trilinear lookups of the whole pyramid. */
typedef struct b200pt_infinite_light {
    int32_t width, height;          /* Lmap->pyramid[0]: uSize(), vSize() (a power of two each after resampling) */
    const float *texels;            /* [height][width][3] RGB texels of level 0                                  */
    float light_to_world[16];       /* Light::LightToWorld.m (row-major)                                         */
    int32_t nu, nv;                 /* Distribution2D: nv conditional rows of nu entries each                    */
    const float *cond_func;         /* [nv][nu]   pConditionalV[v]->func                                         */
    const float *cond_cdf;          /* [nv][nu+1] pConditionalV[v]->cdf                                          */
    const float *cond_func_int;     /* [nv]       pConditionalV[v]->funcInt                                      */
    const float *marg_func;         /* [nv]       pMarginal->func                                                */
    const float *marg_cdf;          /* [nv+1]     pMarginal->cdf                                                 */
    float marg_func_int;            /* pMarginal->funcInt                                                        */
    float power_rgb[3];             /* Lmap->Lookup(Point2f(.5f, .5f), .5f), for Power() (infinite.cpp:86-90)    */
} b200pt_infinite_light;
/* Sets the map and tables of light `light` (kind B200PT_LIGHT_INFINITE) of the scene; the library copies them.  Call it
 * between b200pt_scene_create and b200pt_render_create, once per infinite light. */
int b200pt_scene_set_infinite_light(b200pt_scene *scene, int32_t light, const b200pt_infinite_light *desc);

/* ---- image textures: ImageTexture (textures/imagemap.h) under UVMapping2D (core/texture.cpp:93-99), RGBSpectrum hosts.
 * A MIPMap (core/mipmap.h) is uploaded once as the host built it -- every pyramid level (after the host's power-of-two
 * resampling, "scale" and "gamma"), its wrap mode, filter settings and MIPMap::weightLut -- and bound to any number of
 * (material, parameter) slots, each with its own mapping.  The device filters it with the camera ray's differentials
 * (SurfaceInteraction::ComputeDifferentials, interaction.cpp:103-149) exactly like MIPMap::Lookup(st, dst0, dst1). */
enum { B200PT_WRAP_REPEAT = 0, B200PT_WRAP_BLACK = 1, B200PT_WRAP_CLAMP = 2 };  /* ImageWrap (mipmap.h:47) */
#define B200PT_MIPMAP_MAX_LEVELS 16
typedef struct b200pt_mipmap {
    int32_t n_levels;               /* pyramid.size(): 1 + Log2Int(max(width, height)) of level 0                     */
    int32_t channels;               /* 3 (spectrum texture, RGB texels) or 1 (float texture)                          */
    int32_t width[B200PT_MIPMAP_MAX_LEVELS], height[B200PT_MIPMAP_MAX_LEVELS];  /* uSize(), vSize() of every level:
                                       powers of two, each level max(1, previous / 2)                                  */
    const float *texels[B200PT_MIPMAP_MAX_LEVELS];  /* [height][width][channels] of every level                        */
    int32_t wrap;                   /* B200PT_WRAP_*                                                                  */
    int32_t trilinear;              /* MIPMap::doTrilinear                                                            */
    float max_anisotropy;           /* MIPMap::maxAnisotropy                                                          */
    float weight_lut[128];          /* MIPMap::weightLut                                                              */
} b200pt_mipmap;
/* Material parameter slots a texture can be bound to, and the material types that have them:
 *   KD: matte, plastic   KS: plastic Ks, glass Kr, mirror Kr   KT: glass Kt   ETA, K: metal
 *   ROUGHNESS_U: plastic roughness (both alphas), metal uroughness (or roughness)   ROUGHNESS_V: metal vroughness (or
 *   roughness).  Spectrum slots take 3-channel maps, the roughness slots 1-channel maps. */
enum { B200PT_TEX_KD = 0, B200PT_TEX_KS = 1, B200PT_TEX_KT = 2, B200PT_TEX_ETA = 3, B200PT_TEX_K = 4,
       B200PT_TEX_ROUGHNESS_U = 5, B200PT_TEX_ROUGHNESS_V = 6, B200PT_TEX_SLOTS = 7 };
/* Copies the pyramid to the device; *id names it in b200pt_scene_bind_texture. */
int b200pt_scene_add_mipmap(b200pt_scene *scene, const b200pt_mipmap *desc, int32_t *id);
/* Binds MIPMap `mipmap` with UVMapping2D(su, sv, du, dv) to parameter `slot` of material `material`.  remap_roughness:
 * the material's "remaproughness" (roughness slots only: the looked-up value goes through RoughnessToAlpha). */
int b200pt_scene_bind_texture(b200pt_scene *scene, int32_t material, int32_t slot, int32_t mipmap, float su, float sv,
                              float du, float dv, int32_t remap_roughness);

/* ---- alpha masks: TriangleMesh::alphaMask / shadowAlphaMask (shapes/triangle.cpp:718-743), evaluated inside
 * Triangle::Intersect and IntersectP.  There the texture is looked up without differentials, which for an ImageTexture
 * under UVMapping2D is the bilinear lookup of pyramid level 0 (MIPMap::triangle(0, st)): level 0 is all the device needs.
 * A candidate hit is rejected when a mask is exactly 0 there: closest hits test alpha; any-hit rays (b200pt_trace_any,
 * the path integrator's shadow rays) test alpha and shadowalpha; the volpath integrator's shadow rays test alpha only,
 * as its Tr() intersects with Intersect.  Shape::Pdf and Shape::Sample ignore masks, and so does the device.  Works on
 * RGBSpectrum and SampledSpectrum scenes alike. */
typedef struct b200pt_alpha_mask {
    int32_t width, height;          /* mipmap->pyramid[0]: uSize(), vSize(); 0 x 0 with texels NULL: ConstantTexture(0) */
    const float *texels;            /* [height][width] one float channel                                                 */
    int32_t wrap;                   /* B200PT_WRAP_*                                                                     */
    float su, sv, du, dv;           /* UVMapping2D                                                                       */
} b200pt_alpha_mask;
/* Copies the mask to the device; *id names it in b200pt_scene_set_alpha_masks.  The device keeps each texel as a float4
 * (the layout of the image-texture lookups it shares), 16 bytes per texel: 64 MB for a 2048 x 2048 mask. */
int b200pt_scene_add_alpha_mask(b200pt_scene *scene, const b200pt_alpha_mask *desc, int32_t *id);
/* Per triangle of the scene's numbering (b200pt_scene_desc, n_triangles entries each): the alpha and the shadowalpha
 * mask, or -1; either array may be NULL (no mask of that kind).  A later call replaces the earlier one.  Both entry
 * points must be called before the scene's first trace or b200pt_render_create. */
int b200pt_scene_set_alpha_masks(b200pt_scene *scene, const int32_t *alpha, const int32_t *shadow_alpha);

/* ---- kernel-level entry points (parity tests, traversal benchmarks) -------
 * Replace Scene::Intersect / Scene::IntersectP (core/scene.cpp:45-55) on
 * batches of rays.  `*_dev` variants take device pointers (rays already in
 * HBM); the plain variants copy host buffers in and out. */
int b200pt_trace_closest(b200pt_scene *scene, const b200pt_ray *rays, b200pt_hit *hits, int64_t n);
int b200pt_trace_any(b200pt_scene *scene, const b200pt_ray *rays, uint8_t *occluded, int64_t n);
int b200pt_trace_closest_dev(b200pt_scene *scene, uint64_t rays_dev, uint64_t hits_dev, int64_t n);
int b200pt_trace_any_dev(b200pt_scene *scene, uint64_t rays_dev, uint64_t occluded_dev, int64_t n);

/* ---- render: replaces SamplerIntegrator::Render (integrator.cpp:228-339) -- */
int b200pt_render_create(b200pt_scene *scene, const b200pt_camera_desc *camera,
                         const b200pt_film_desc *film, const b200pt_sampler_desc *sampler,
                         const b200pt_integrator_desc *integrator, b200pt_render **out);
void b200pt_render_destroy(b200pt_render *r);

/* Number of 16x16 tiles in x and y (integrator.cpp:235-237). */
int b200pt_render_tile_counts(const b200pt_render *r, int32_t *nx, int32_t *ny);

/* Film::Clear (film.cpp:108-115) on the device film. */
int b200pt_film_clear(b200pt_render *r);

/* Renders the given tiles (tile index = y*nx + x, the reference's `seed`,
 * integrator.cpp:247) with ALL samples per pixel and merges them into the
 * device film (raw XYZ sums + filter weight sums, film.cpp:117-130).
 * tiles == NULL renders tiles [0, n_tiles) in order.  Asynchronous on the
 * context's stream: argument errors are returned here, a failure of the
 * device work itself (a CUDA error inside a launch) is reported by the next
 * call that synchronises -- b200pt_ctx_synchronize, b200pt_film_read_*,
 * b200pt_get_stats -- as B200PT_ERR_CUDA with b200pt_last_error() naming it.
 * Dropped traversal-stack pushes and sampler-dimension overruns are counted,
 * never silent (b200pt_stats::stack_overflows / dimension_overflows). */
int b200pt_render_tiles(b200pt_render *r, const int32_t *tiles, int64_t n_tiles);

/* Device address and size of the film accumulation buffer: float4 per cropped
 * pixel = (X, Y, Z, filterWeightSum), row-major over cropped_bounds.  This is
 * the buffer a multi-GPU caller reduces (sum) across ranks before read-back. */
int b200pt_film_device_buffer(b200pt_render *r, uint64_t *dev_ptr, uint64_t *n_floats);

/* Copies the raw film (X,Y,Z,weight per pixel) to the host (synchronises). */
int b200pt_film_read_raw(b200pt_render *r, float *xyzw);

/* ---- multi-GPU film merge ------------------------------------------------
 * One process per GPU renders a disjoint set of tiles of the SAME film (full-film sampler, SURVEY 8e); the raw
 * (X,Y,Z,weight) sums are then added on `root` with one ncclReduce over NVLink.  This replaces what the reference's
 * distributed runs do with files afterwards (imgtool assemble, tools/imgtool.cpp:190-285) and the MergeFilmTile
 * mutex inside one process (film.cpp:117-130).  NCCL is loaded at run time (libnccl.so.2; B200PT_NCCL_LIB overrides).
 *
 * b200pt_comm_create: bootstraps a communicator of `world_size` processes through a file every rank can reach:
 * rank 0 writes the NCCL unique id to `id_file`, the others wait for it (up to 120 s).  b200pt_comm_from_nccl wraps
 * a communicator the host application already owns (an ncclComm_t passed as void *; it is not destroyed). */
typedef struct b200pt_comm b200pt_comm;
int b200pt_comm_create(b200pt_ctx *ctx, int rank, int world_size, const char *id_file, b200pt_comm **out);
int b200pt_comm_from_nccl(b200pt_ctx *ctx, void *nccl_comm, int rank, int world_size, b200pt_comm **out);
void b200pt_comm_destroy(b200pt_comm *comm);
/* Adds the raw film sums of all ranks into `root`'s film buffer (in place, on the context's stream; the other
 * ranks' buffers keep their own partial sums).  Every rank of the communicator must call it. */
int b200pt_film_reduce(b200pt_render *r, b200pt_comm *comm, int root);
/* Film::WriteImage's pixel pipeline (film.cpp:174-203): XYZ->RGB, divide by
 * weight, clamp >=0, *scale; rgb is [h][w][3] over the cropped bounds. */
int b200pt_film_read_rgb(b200pt_render *r, float *rgb);

/* Diagnostics for parity tests: the Sobol' sample values the device generates
 * for (pixel, sample index, dimension range) -- GlobalSampler::Get1D stream,
 * sampler.cpp:181-195 -- and the camera rays of the first `n` samples of a
 * pixel (RayDifferential main ray only). */
int b200pt_debug_sobol(b200pt_render *r, int32_t px, int32_t py, int64_t sample, int32_t dim0,
                       int32_t n_dims, float *out);
int b200pt_debug_camera_rays(b200pt_render *r, int32_t px, int32_t py, int32_t n_samples,
                             b200pt_ray *out);
/* Per-sample radiance (after the NaN / negative / infinite guards of
 * integrator.cpp:294-315) of one pixel: out is [samples_per_pixel][3]. */
int b200pt_debug_pixel_samples(b200pt_render *r, int32_t px, int32_t py, float *out_rgb);

/* Options: "instrument" (count BVH nodes fetched / triangles tested in the
 * traversal kernels -- the algorithmic-bytes figure of the roofline) and
 * "profile" (bracket every launch with CUDA events on the context's stream so
 * b200pt_get_stats reports device time per kernel class). Both default to 0. */
int b200pt_render_set_option(b200pt_render *r, const char *name, int value);

int b200pt_get_stats(b200pt_render *r, b200pt_stats *out);
int b200pt_reset_stats(b200pt_render *r);

/* ---- host helpers (no device work) ---------------------------------------
 * Mirror of the host-side math a caller outside pbrt needs to fill the
 * descriptors exactly like the reference would:
 *  - camera matrices from LookAt + Perspective(fov, 1e-2, 1000) + screen
 *    window, as ProjectiveCamera does (core/camera.h:84-115,
 *    core/transform.cpp:203-249,303-318, cameras/perspective.cpp:227-273);
 *  - TrowbridgeReitzDistribution::RoughnessToAlpha (microfacet.h:123-128). */
int b200pt_host_perspective_camera(const float eye[3], const float look[3], const float up[3],
                                   float fov_degrees, int32_t xres, int32_t yres,
                                   b200pt_camera_desc *out);
float b200pt_host_roughness_to_alpha(float roughness);
/* OrenNayar's A and B from sigma in degrees (reflection.h:414-420), clamped like matte.cpp:54 */
void b200pt_host_oren_nayar(float sigma_degrees, float *A, float *B);
/* CreateSpotLight (spot.cpp:104-124) at the identity CTM: fills kind, position, the cone cosines and world_to_light. */
void b200pt_host_spot_light(const float from[3], const float to[3], float coneangle, float conedelta,
                            b200pt_area_light *out);
/* Sphere constructor (sphere.h:49-61): out = {zMin, zMax, thetaMin, thetaMax, phiMax}. */
void b200pt_host_sphere_params(float radius, float zmin, float zmax, float phimax_degrees, float out[5]);

#ifdef __cplusplus
}
#endif
#endif /* B200PT_H */
