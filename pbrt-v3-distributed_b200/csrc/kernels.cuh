// kernels.cuh -- device-side data layout shared by kernels.cu and api.cu.
//
// Wavefront organisation of SamplerIntegrator::Render (integrator.cpp:228-339):
// a *batch* is a set of 16x16 film tiles rendered with all their samples at
// once.  Path slot = ((tile_in_batch * 256 + pixel_in_tile) * spp + sample),
// i.e. the reference's loop nest tile -> pixel (row-major) -> sample flattened,
// so a warp holds 32 consecutive samples of one pixel (coherent camera rays)
// and the film kernel can re-create the reference's per-tile summation order.
// Per-slot state lives in two 128-byte records per slot (PathRec, DirectRec);
// queues of slot indices connect the stages.
#ifndef B200PT_KERNELS_CUH
#define B200PT_KERNELS_CUH

#include <cuda_runtime.h>

#include "wbvh_traverse.cuh"
#include "pt_core.cuh"
#include "pt_sphere.cuh"

namespace B200PT_NS {

struct DevLight {
    uint32_t tri;  // leaf-order triangle index, or SPHERE_HIT_BASE | sphere index (the id traversal reports)
    float lemit[3];
    int two_sided;
    float area;  // Triangle::Area(), computed on the host
    // delta lights (b200pt_area_light::kind != 0): position = pLight or wLight, the spot's cone and WorldToLight,
    // the distant light's 2 * worldRadius
    int kind;
    float position[3];
    float cos_total_width, cos_falloff_start;
    float world_to_light[16];
    float two_world_radius;
};

struct DevScene {
    const U4 *nodes;
    const uint32_t *tri_base;  // per node: first triangle of its leaf children (wbvh.h)
    const uint8_t *lut;        // permute_slots table (B200PT_LUT_BYTES)
    TravBounds bounds;         // padded bounds of the top-level tree
    const F4 *tris;
    const b200pt_material *materials;
    const float *material_spectra;  // SampledSpectrum build: [n_materials][5][60] (kd, ks, kt, eta, k), else nullptr
    uint32_t n_nodes, n_tris;
    const F4 *tri_n;   // optional per-vertex shading normals, 3 x float4 per triangle (leaf order)
    const F4 *tri_uv;  // optional uvs, 2 x float4 per triangle: (u0 v0 u1 v1) (u2 v2 - -)
    const DevSphere *spheres;  // Sphere shapes, tested outside the BVH (k_spheres)
    uint32_t n_spheres;
    const DevInstance *instances;  // object instances, tested by the same pass; their BVHs follow the top-level one
    uint32_t n_instances;
    uint32_t tlas_node_off, tlas_tri_off;  // 8-wide tree over the instances' leaf boxes (its "triangles" name instances), 0 = none
};

// queue ids inside one bounce's counter block
enum { Q_PATH = 0, Q_MAT0 = 1, Q_SHADOW = 5, Q_MIS = 6, Q_NEXT = 7, Q_PER_BOUNCE = 8 };
// meta word of a path: dim (16 bits) | bounces (8) | flags (8)
enum { PF_SPECULAR = 1 };
// pending direct-lighting flags
enum { PEND_LIGHT = 1, PEND_BSDF = 2 };

// Per-slot state.  Every kernel after raygen reaches its slots through a queue, so the slots a warp touches are scattered
// and each access costs whole 32-byte sectors.  The state is therefore kept in two records of four sectors per slot:
// a sector holds fields of one slot only, the fields one kernel uses together share a sector, and a kernel that rewrites
// a sector writes all of it where it has the values.  Both records are 128 bytes, so one stride indexes either.
// SampledSpectrum build: the float4 spectra (beta, L, A, B, beta_ld) keep only their fourth component; the 60 bins live in
// the slot-major RenderDev::s_* arrays.
struct alignas(128) PathRec {
    float4 o;            // [0] ray origin, etaScale             the traversal fetches the ray as this one sector
    float4 d;            //     ray direction, meta (bits)
    float4 beta;         // [1] beta.rgb, 0
    float4 L;            //     L.rgb, bleed code (bits)
    uint64_t sobol;      // [2] Sobol' index of (pixel, sample)
    uint32_t hit;        //     closest-hit triangle (leaf order) of the path ray
    uint32_t hit_inst;   //     instance of that hit when the triangle belongs to an object (scenes with instances)
    uint32_t unused[12];
};
struct alignas(128) DirectRec {
    float4 sh_o;         // [0] shadow ray origin, light number (bits)     the any-hit traversal's ray
    float4 sh_d;         //     shadow ray direction, pending flags (bits)
    float4 mi_o;         // [1] MIS (BSDF-sampled) ray origin, scattering pdf   the MIS traversal's ray
    float4 mi_d;         //     MIS ray direction
    float4 A;            // [2] light-sampling term f*Li*w/lightPdf
    float4 B;            //     BSDF-sampling term f*Le*w/scatteringPdf, valid if the MIS ray reaches the light
    float4 beta_ld;      // [3] beta at the time of the direct-lighting estimate, light pick pdf
    uint32_t mis_hit;    //     closest-hit triangle of the MIS ray
    uint8_t occluded;    //     any-hit result of the shadow ray
    uint8_t unused[11];
};
static_assert(sizeof(PathRec) == 128 && sizeof(DirectRec) == 128, "per-slot records are four 32-byte sectors");
// float4 stride of the ray pairs (PathRec::o/d, DirectRec::sh_o/sh_d, DirectRec::mi_o/mi_d) from one slot to the next
constexpr int REC_F4 = (int)(sizeof(PathRec) / sizeof(float4));

struct RenderDev {
    DevScene scene;
    SamplerParams sampler;
    CameraParams camera;
    // film
    int crop[4];            // cropped pixel bounds
    int pixel_bounds[4];    // integrator "pixelbounds"
    float max_sample_luminance;
    float4 *film;           // [h][w] (X, Y, Z, weight) raw sums
    // general pixel filter (film.h:121-161); filter_general == 0 selects the box-radius-0.5 path
    int filter_general;
    float filter_radius[2], filter_inv_radius[2];
    int apron[2];                   // FilmTile pixels beyond the 16x16 tile on each side (film.cpp:95-106)
    const float *filter_table;      // [16][16] Film::filterTable
    float2 *pfilm;                  // per slot: CameraSample::pFilm (general filter only)
    float4 *tile_film;              // [tiles_per_batch][16 + 2 apron_y][16 + 2 apron_x] merged tile sums (XYZ, weight)
    int32_t *tile_slot;             // [tiles_x * tiles_y] position of a tile in the current batch or -1
    // integrator
    int max_depth;
    float rr_threshold;
    // lights + Distribution1D of the chosen strategy
    const DevLight *lights;
    int n_lights;
    const float *light_cdf;   // [n_lights + 1]
    const float *light_func;  // [n_lights]
    float light_func_int;
    int has_delta_lights;     // some light is a point / spot / distant light (handled by the full shading variant)
    // SpatialLightDistribution: per-voxel func [n_lights], cdf [n_lights+1], funcInt
    SpatialGrid grid;
    float *sp_func, *sp_cdf, *sp_func_int;
    // batch
    int tiles_x, tiles_y;
    const int32_t *tile_list;  // tile ids of the whole render_tiles call
    uint32_t capacity;         // path slots per batch
    // per-slot state
    PathRec *path;
    DirectRec *direct;
    // SampledSpectrum build only (nullptr otherwise): the bins of beta, L, A, B and beta_ld, slot-major [capacity][60]
    // (240 contiguous bytes per slot, see ld_spec); the float4 fields of the records then keep just their fourth component
    float *s_beta, *s_L, *s_A, *s_B, *s_beta_ld;
    const float *light_spectra;  // [n_lights][60]: Lemit / I / L of each light
    uint8_t *pix_bleed;  // [tiles_per_batch*256] pixel has a sample whose box-filter footprint leaves the pixel
    // queues (slot indices) and their counters
    uint32_t *q_path[2];       // ping-pong
    uint32_t *q_mat[4];
    uint32_t *q_shadow;
    uint32_t *q_mis;
    uint32_t *q_sorted;        // queue re-ordered by (ray octant, Morton cell of the origin)
    uint32_t *sort_keys;       // key per queue entry
    uint32_t *sort_hist;       // [SORT_BUCKETS] counting-sort histogram / cursors
    float sort_lo[3], sort_inv[3];  // origin -> 32^3 grid over the scene bounds
    uint32_t *qcount;          // [(max_depth + 2) * Q_PER_BOUNCE]
    uint32_t *work;            // persistent-fetch counters, one per launch of a batch
    unsigned long long *stats; // camera, regular, shadow, nodes, tris
    // VolPathIntegrator (b200pt_integrator_desc::volumetric / medium): light sampling at every vertex; with has_medium
    // every ray is inside one homogeneous medium (RGB build only)
    int volpath, has_medium;
    float med_sigma_s[3], med_sigma_t[3], med_g;
    const float *med_spectra;  // SampledSpectrum build: [2][60] = sigma_s, sigma_t (else the two arrays above)
    // Media bounded by null-material spheres (b200pt_integrator_desc::bounded_media, RGB build): medium ids are -1 = vacuum,
    // 0 = the medium around the scene, k >= 1 = bounded_media[k - 1].  The path ray's medium is per-slot state; rays that
    // reach a boundary are traced again from the far side within the same bounce (q_cross), shadow and MIS rays walk from
    // boundary to boundary while their transmittance accumulates (k_shadow_walk / k_mis_walk).
    int med_general;
    const float *media_tab;    // [1 + n_bounded][2][3] = sigma_s, sigma_t of medium id k
    const float *media_g;      // [1 + n_bounded]
    const int32_t *sphere_med; // [n_spheres] medium id inside a boundary sphere, -1 for an ordinary sphere
    int32_t *cur_med;          // per slot: medium of the path ray
    uint32_t *q_cross[2];      // path rays that crossed a boundary (ping-pong between passes of one bounce)
    uint32_t *q_walk[2];       // shadow / MIS rays that crossed a boundary
    uint32_t *sh_hit;          // closest hit of the shadow ray's current segment
    float4 *A2;                // pending light sample: Li, lightPdf   (A then holds f, MIS weight; weight < 0: delta light)
    float4 *sh_tr, *mi_tr;     // transmittance so far along the shadow / MIS ray, medium id of the current segment (bits)
    float4 *sh_p1, *sh_p1e, *sh_p1n;  // the light sample the shadow ray is re-aimed at after each boundary (SpawnRayTo)
    unsigned long long *dim_overflows;  // paths ended because their sampler dimension ran past the host's tables
};

// resident CTAs of k_trace per SM (128 threads each).  7 (up to 72 registers, no spills) measured fastest on the H100
// (cfg4, 16 batches, profiles/README.md): +3 % over 8 (64 registers, a few spilled per-ray constants) and +1.5 % over 6.
#ifndef B200PT_TRACE_CTAS
#define B200PT_TRACE_CTAS 7
#endif

struct TraceArgs {
    const U4 *nodes;
    const uint32_t *tri_base;  // parallel to nodes
    const uint8_t *lut;        // permute_slots table in global memory (k_trace stages it in shared memory)
    TravBounds bounds;         // padded bounds of the top-level tree
    TravBounds tlas_bounds;    // ... of the tree over the instances' leaf boxes
    const F4 *tris;
    const float4 *ray_o;   // o.xyz (+ t_max in .w when t_max_from_w)
    const float4 *ray_d;
    const uint32_t *queue; // slot indices or nullptr for identity
    const uint32_t *count; // device-side number of rays
    uint32_t *work;        // persistent fetch counter (zeroed)
    float fixed_t_max;     // used unless t_max_from_w
    int t_max_from_w;
    int stride;            // ray_o/ray_d element stride in float4 (REC_F4 for the per-slot records, 2 for b200pt_ray)
    uint32_t *hit_out;     // closest: triangle per slot
    b200pt_hit *full_out;  // closest: optional full record (prim id, t, b0, b1)
    uint8_t *occ_out;      // any-hit result per slot
    int out_stride;        // bytes from one slot's hit_out / hit_inst_out / occ_out entry to the next (see slot_out)
    // classification of closest hits by material family
    uint32_t *q_mat[4];
    uint32_t *qcount_mat;  // &qcount[bounce*Q_PER_BOUNCE + Q_MAT0]
    const b200pt_material *materials;
    unsigned long long *stats;  // nodes/tris counters when instrumented
    int ctas;                   // resident CTAs per SM the launch is compiled for (B200PT_TRACE_CTAS, 6 or 8), 0 = default
    uint32_t n_staged;          // > 0: k_trace copies nodes [0, n_staged) -- the top of the breadth-first tree -- into shared
                                // memory with one TMA bulk copy (cp.async.bulk + mbarrier) and reads them there
    int refill_lanes;           // refill the warp when fewer lanes than this are still traversing
    int postpone_pct;           // triangle postponing threshold (% of converged lanes), 0 = off
    uint32_t magic;             // 0x47000000 as a run-time value (PRMT's second source stays in a register, see plane_2p15)
    // sphere pass (launch_spheres): same rays, after the traversal launch
    const DevSphere *spheres;
    uint32_t n_spheres;
    uint32_t n_tris;            // sphere k is reported as primitive n_tris + k in full_out
    uint32_t *sphere_work;      // persistent fetch counter of the sphere pass (zeroed)
    int sphere_refill_lanes;    // the sphere / instance pass refills a warp when fewer lanes than this are still walking
    const DevInstance *instances;
    uint32_t n_instances;
    uint32_t tlas_node_off, tlas_tri_off;  // see DevScene
    uint32_t *hit_inst_out;     // instance of an object-triangle hit (closest, render path)
};
// the entry of `slot` in a traversal output: a field of the per-slot records or an element of a plain array
template <class T>
__device__ __forceinline__ T &slot_out(T *base, uint32_t slot, int stride) {
    return *reinterpret_cast<T *>(reinterpret_cast<char *>(base) + (size_t)slot * (size_t)stride);
}

void launch_raygen(const RenderDev *dev, uint32_t batch_first_tile, uint32_t n_batch_tiles, uint32_t n_slots,
                   cudaStream_t s);
// grid = SMs of the device (the launcher multiplies by the CTAs per SM of the chosen variant)
void launch_trace(const TraceArgs &a, bool any_hit, bool classify, bool count, int n_sm, cudaStream_t s);
// Scenes with object instances (and a tree over them): top-level triangles + instances in one persistent two-level
// traversal (k_trace2); launch_spheres is then only needed for Sphere shapes.  Not part of the CPU check build.
void launch_trace2(const TraceArgs &a, bool any_hit, bool classify, int n_sm, cudaStream_t s);
// Tests the spheres against the rays of a finished traversal launch (tMax shortened by the triangle hit),
// updates hit_out / full_out / occ_out and, with `classify`, appends the slots to the BSDF-family queues
// (the traversal launch then runs without classification).
void launch_spheres(const TraceArgs &a, bool any_hit, bool classify, int grid, cudaStream_t s);
void launch_shade(const RenderDev *dev, int material, bool vertex_data, int bounce, uint32_t *work, int grid,
                  cudaStream_t s);
void launch_resolve(const RenderDev *dev, int bounce, uint32_t *work, int grid, cudaStream_t s);
// Medium pass of a bounce (scenes inside a homogeneous medium): after the closest-hit launch, before the shading kernels.
void launch_medium(const RenderDev *dev, int bounce, uint32_t *work, int grid, cudaStream_t s);
// Scenes with bounded media: one pass of the medium kernel over `queue` (the bounce's path queue, then the rays that crossed
// a boundary); crossers of this pass are appended to q_cross[out] / *cross_count.  count_rays: add the pass's rays to the
// regular-ray counter (every pass but a bounce's first, which the queue counters already cover).
void launch_medium_general(const RenderDev *dev, const RenderDev &host, int bounce, const uint32_t *queue, const uint32_t *count,
                           int out, uint32_t *cross_count, uint32_t *work, bool count_rays, int grid, cudaStream_t s);
// One segment of the shadow (any = false: MIS) rays' walk through the boundaries: reads the segment's closest hit, ends the
// ray (occluded / A or mis_hit / B final) or re-queues it behind the boundary into q_walk[out] / *walk_count.
void launch_direct_walk(const RenderDev *dev, const RenderDev &host, bool shadow, const uint32_t *queue, const uint32_t *count,
                        int out, uint32_t *walk_count, uint32_t *work, bool count_rays, int grid, cudaStream_t s);
#define SORT_BUCKETS (1u << 18)  // 3 octant bits + 15 Morton bits
// Counting sort of a queue of slots by the coherence key of the rays they refer to; `out` receives
// the permuted queue (order inside a bucket is arbitrary -- it never affects a path's arithmetic).
// ray_o / ray_d point at the ray pair of slot 0 in the per-slot records (stride REC_F4).
void launch_sort_queue(const RenderDev *dev, const RenderDev &host, const uint32_t *queue, const uint32_t *count,
                       const float4 *ray_o, const float4 *ray_d, int grid, cudaStream_t s);
void launch_sobol_table(const uint32_t *mat32, uint32_t *table, int n_dims, cudaStream_t s);
// Fills the per-voxel light distributions (all voxels, once per render object).
void launch_spatial_build(const RenderDev *dev, const RenderDev &host, cudaStream_t s);
void launch_film(const RenderDev *dev, uint32_t batch_first_tile, uint32_t n_batch_tiles, cudaStream_t s);
// General pixel filter: per-tile FilmTile sums in the reference's sample order, then the tiles of the batch are
// merged into the film in tile-list order (Film::MergeFilmTile order of a single-threaded reference run).
void launch_film_general(const RenderDev *dev, const RenderDev &host, uint32_t batch_first_tile, uint32_t n_batch_tiles,
                         cudaStream_t s);
void launch_accumulate_stats(const RenderDev *dev, uint32_t n_camera, cudaStream_t s);
void launch_debug_sobol(const RenderDev *dev, int px, int py, long long sample, int dim0, int n, float *out,
                        cudaStream_t s);
void launch_debug_camera(const RenderDev *dev, int px, int py, int n, b200pt_ray *out, cudaStream_t s);
void launch_film_rgb(const float4 *film, float *rgb, int n_pixels, float scale, cudaStream_t s);

}  // namespace B200PT_NS
#endif
