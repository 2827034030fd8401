// kernels.cu -- the sm_90a kernels of the wavefront path tracer.
//
//   k_raygen   K1  Sobol' camera samples -> camera rays (GetCameraSample + GenerateRayDifferential)
//   k_trace    K2/K3  persistent-thread closest-hit / any-hit traversal of the 7-wide BVH (wbvh.h); the
//              closest-hit epilogue classifies hits into per-material-family queues
//              (warp-ballot aggregated appends)
//   k_shade<M> K4  one kernel per BSDF family: surface reconstruction, emission, light
//              sampling + MIS bookkeeping (EstimateDirect), BSDF sampling, Russian roulette
//   k_resolve      adds the direct-lighting estimate once shadow / MIS rays are traced
//   k_film     K6  FilmTile::AddSample + MergeFilmTile in the reference's summation order
// All kernels of a batch run back to back on one stream with device-side queue
// counters; the host never synchronises inside a batch.
#include <cstdio>

#include "kernels.cuh"
#include "pt_texture.cuh"

namespace B200PT_NS {

#define FULL_MASK 0xffffffffu

__device__ __forceinline__ V3 v3(const float4 &f) { return mk(f.x, f.y, f.z); }
__device__ __forceinline__ V3 v3(const F4 &f) { return mk(f.x, f.y, f.z); }
__device__ __forceinline__ float4 f4(const V3 &v, float w) { return make_float4(v.x, v.y, v.z, w); }
// A per-slot spectrum travels with one packed scalar.  RGBSpectrum build: one float4 of a record (r, g, b, w).
// SampledSpectrum build: the float4 keeps only w and the 60 bins live slot-major in a second array, [capacity][60] (240
// contiguous bytes per slot, read and written as float4s).  A [bin][capacity] layout would coalesce only if a warp's slots
// were neighbours; the slots of a BSDF family's queue are scattered, so every 4-byte access would cost a 32-byte sector.
__device__ __forceinline__ Spec ld_spec(const float4 &f, const float *bins, uint32_t slot, float *w) {
    *w = f.w;
#if B200PT_NSPEC == 3
    (void)bins;
    (void)slot;
    return rgb(f.x, f.y, f.z);
#else
    Spec s;
    const float4 *p4 = reinterpret_cast<const float4 *>(bins + (size_t)slot * B200PT_NSPEC);
#pragma unroll
    for (int q = 0; q < B200PT_NSPEC / 4; ++q) {
        const float4 v = p4[q];
        s.c[4 * q] = v.x;
        s.c[4 * q + 1] = v.y;
        s.c[4 * q + 2] = v.z;
        s.c[4 * q + 3] = v.w;
    }
    return s;
#endif
}
__device__ __forceinline__ void st_spec(float4 &f, float *bins, uint32_t slot, const Spec &s, float w) {
#if B200PT_NSPEC == 3
    (void)bins;
    (void)slot;
    f = make_float4(s.c[0], s.c[1], s.c[2], w);
#else
    f = make_float4(0.f, 0.f, 0.f, w);
    float4 *p4 = reinterpret_cast<float4 *>(bins + (size_t)slot * B200PT_NSPEC);
#pragma unroll
    for (int q = 0; q < B200PT_NSPEC / 4; ++q) p4[q] = make_float4(s.c[4 * q], s.c[4 * q + 1], s.c[4 * q + 2], s.c[4 * q + 3]);
#endif
}
// Shading writes beta_ld's sector whole: the traversal results beside it are reset with one 16-byte store (the shadow and
// MIS launches of the bounce overwrite them before anything reads them).
__device__ __forceinline__ void reset_direct_hits(DirectRec &D) {
    *reinterpret_cast<float4 *>(&D.mis_hit) = make_float4(__uint_as_float(B200PT_MISS), 0.f, 0.f, 0.f);
}
__device__ __forceinline__ void st_beta_ld(DirectRec &D, float *bins, uint32_t slot, const Spec &beta, float pickPdf) {
    st_spec(D.beta_ld, bins, slot, beta, pickPdf);
    reset_direct_hits(D);
}
// Lemit / I / L of light `lightNum` (b200pt_area_light::lemit, or its row of b200pt_scene_desc::light_spectra)
__device__ __forceinline__ Spec light_emit(const RenderDev *R, int lightNum, const DevLight &l) {
#if B200PT_NSPEC == 3
    (void)R;
    (void)lightNum;
    return rgbp(l.lemit);
#else
    (void)l;
    return rgbp(R->light_spectra + (size_t)lightNum * B200PT_NSPEC);
#endif
}

// sigma_s / sigma_t of the medium around the scene (RenderDev::med_*)
__device__ __forceinline__ Spec medium_sigma_s(const RenderDev *R) {
#if B200PT_NSPEC == 3
    return rgbp(R->med_sigma_s);
#else
    return rgbp(R->med_spectra);
#endif
}
// media bounded by surfaces (RGB build): coefficients of medium id k (RenderDev::media_tab)
__device__ __forceinline__ Spec media_sigma_s(const RenderDev *R, int k) { return rgbp(R->media_tab + (size_t)k * 2 * B200PT_NSPEC); }
__device__ __forceinline__ Spec media_sigma_t(const RenderDev *R, int k) { return rgbp(R->media_tab + ((size_t)k * 2 + 1) * B200PT_NSPEC); }
__device__ __forceinline__ Spec medium_sigma_t(const RenderDev *R) {
#if B200PT_NSPEC == 3
    return rgbp(R->med_sigma_t);
#else
    return rgbp(R->med_spectra + B200PT_NSPEC);
#endif
}

#ifdef B200PT_HOST_EMU
// CPU check build (tests/emu): threads run one after the other, so a "warp" is one lane
__device__ __forceinline__ uint32_t warp_append(uint32_t *counter, bool pred) { return pred ? atomicAdd(counter, 1u) : 0u; }
__device__ __forceinline__ bool warp_fetch(uint32_t *work, uint32_t n, uint32_t *item) {
    const uint32_t base = atomicAdd(work, 1u);
    if (base >= n) return false;
    *item = base;
    return true;
}
#else
// Warp-aggregated append: every lane of the warp must call it (converged);
// lanes with pred get consecutive positions behind one atomicAdd.
__device__ __forceinline__ uint32_t warp_append(uint32_t *counter, bool pred) {
    const uint32_t mask = __ballot_sync(FULL_MASK, pred);
    if (mask == 0) return 0;
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(mask) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(counter, (uint32_t)__popc(mask));
    base = __shfl_sync(FULL_MASK, base, leader);
    return base + (uint32_t)__popc(mask & ((1u << lane) - 1u));
}

// Persistent-thread fetch of 32 work items per warp.
__device__ __forceinline__ bool warp_fetch(uint32_t *work, uint32_t n, uint32_t *item) {
    const int lane = threadIdx.x & 31;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(work, 32u);
    base = __shfl_sync(FULL_MASK, base, 0);
    if (base >= n) return false;
    *item = base + (uint32_t)lane;
    return true;
}

#endif  // B200PT_HOST_EMU

// per-vertex shading data of triangle `ti` (flags: bit 18 = normals, bit 19 = uvs)
// VTX = false is the variant for scenes without any per-vertex data: the defaults fold to constants.
template <bool VTX>
__device__ __forceinline__ void load_shading(const DevScene &sc, uint32_t ti, uint32_t mflags, TriShading *t) {
    default_shading(t);
    if (!VTX) return;
    if (mflags & B200PT_TRI_HAS_NORMALS) {
        const F4 *np = sc.tri_n + (size_t)ti * 3;
        t->has_n = 1;
        t->n0 = v3(ld_f4(np));
        t->n1 = v3(ld_f4(np + 1));
        t->n2 = v3(ld_f4(np + 2));
    }
    if (mflags & B200PT_TRI_HAS_UVS) {
        const F4 a = ld_f4(sc.tri_uv + (size_t)ti * 2), b = ld_f4(sc.tri_uv + (size_t)ti * 2 + 1);
        t->uv[0] = a.x;
        t->uv[1] = a.y;
        t->uv[2] = a.z;
        t->uv[3] = a.w;
        t->uv[4] = b.x;
        t->uv[5] = b.y;
    }
}

// ---- classification of closest hits, shared by the traversal kernels and the medium passes
// BSDF family (the queue, the k_shade instance) of a hit with material word `mflags`
__device__ __forceinline__ int hit_family(const b200pt_material *materials, uint32_t mflags) { return materials[mflags & 0xffffu].type; }
// Appends `slot` to the queue of BSDF family `family` (-1: to none).  Every lane of the warp must call it (converged).
__device__ __forceinline__ void append_family(uint32_t *const *q_mat, uint32_t *qcount_mat, int family, uint32_t slot) {
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        const bool mine = family == m;
        const uint32_t pos = warp_append(&qcount_mat[m], mine);
        if (mine) q_mat[m][pos] = slot;
    }
}

// ------------------------------------------------------------------ tile maths
struct TileRect {
    int x0, y0, x1, y1;  // sample-space rectangle of the tile (integrator.cpp:251-255)
};
__device__ __forceinline__ TileRect tile_rect(const RenderDev *R, int tile) {
    TileRect t;
    const int tx = tile % R->tiles_x, ty = tile / R->tiles_x;
    t.x0 = R->sampler.sb[0] + tx * 16;
    t.x1 = min(t.x0 + 16, R->sampler.sb[2]);
    t.y0 = R->sampler.sb[1] + ty * 16;
    t.y1 = min(t.y0 + 16, R->sampler.sb[3]);
    return t;
}
// a pixel of the tile is rendered iff it lies in the tile and in "pixelbounds" (integrator.cpp:273)
__device__ __forceinline__ bool pixel_rendered(const RenderDev *R, const TileRect &t, int px, int py) {
    return px >= t.x0 && px < t.x1 && py >= t.y0 && py < t.y1 && px >= R->pixel_bounds[0] &&
           px < R->pixel_bounds[2] && py >= R->pixel_bounds[1] && py < R->pixel_bounds[3];
}

// ---------------------------------------------------------------------- raygen
// PFILM: keep pFilm for every sample, not only under a general filter (textured scenes rebuild the camera ray's differentials)
template <bool PFILM>
__device__ __forceinline__ void raygen(const RenderDev *R, uint32_t first_tile, uint32_t n_slots) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    bool valid = false;
    if (slot < n_slots) {
        const uint32_t spp = (uint32_t)R->sampler.spp;
        const uint32_t sample = slot % spp;
        const uint32_t pix = (slot / spp) & 255u;
        const uint32_t tb = slot / (spp * 256u);
        const int tile = R->tile_list[first_tile + tb];
        const TileRect t = tile_rect(R, tile);
        const int px = t.x0 + (int)(pix & 15u), py = t.y0 + (int)(pix >> 4);
        if (pixel_rendered(R, t, px, py)) {
            valid = true;
            const SamplerParams &sp = R->sampler;
            SobolStream st;
            st.index = sampler_index(sp, sample, px, py);
            st.dim = 0;
            st.px = px;
            st.py = py;
            float u[2], ul[2];
            get2d(sp, st, u);  // sampler.cpp:46-52
            float pFilm[2] = {(float)px + u[0], (float)py + u[1]};
            (void)get1d(sp, st);  // time
            get2d(sp, st, ul);
            V3 o, d;
            float tMax;
            generate_camera_ray(R->camera, pFilm, ul, &o, &d, &tMax);
            // box-filter footprint of the sample (film.h:126-132, radius 0.5)
            const float dx = pFilm[0] - 0.5f, dy = pFilm[1] - 0.5f;
            uint32_t code = 0;
            if ((int)ceilf(dx - 0.5f) < px) code |= 1u;
            if ((int)floorf(dx + 0.5f) + 1 > px + 1) code |= 2u;
            if ((int)ceilf(dy - 0.5f) < py) code |= 4u;
            if ((int)floorf(dy + 0.5f) + 1 > py + 1) code |= 8u;
            if (code) R->pix_bleed[tb * 256u + pix] = 1;
            if (PFILM || R->filter_general) R->pfilm[slot] = make_float2(pFilm[0], pFilm[1]);
            PathRec &P = R->path[slot];
            P.o = f4(o, 1.f);                                // etaScale = 1
            P.d = f4(d, __uint_as_float((uint32_t)st.dim));  // dim = 5, bounces = 0, flags = 0
            st_spec(P.beta, R->s_beta, slot, rgb1(1.f), 0.f);
            st_spec(P.L, R->s_L, slot, rgb1(0.f), __uint_as_float(code));
            P.sobol = st.index;
            DirectRec &D = R->direct[slot];  // no direct lighting pending
            D.sh_o = make_float4(0.f, 0.f, 0.f, 0.f);
            D.sh_d = make_float4(0.f, 0.f, 0.f, 0.f);
            if (R->med_general) R->cur_med[slot] = R->has_medium ? 0 : -1;  // the camera's medium (camera.h:76)
        }
    }
    const uint32_t pos = warp_append(&R->qcount[Q_PATH], valid);
    if (valid) R->q_path[0][pos] = slot;
}
__global__ void __launch_bounds__(256) k_raygen(const RenderDev *R, uint32_t first_tile, uint32_t n_slots) {
    raygen<false>(R, first_tile, n_slots);
}
#if B200PT_NSPEC == 3
__global__ void __launch_bounds__(256) k_raygen_pfilm(const RenderDev *R, uint32_t first_tile, uint32_t n_slots) {
    raygen<true>(R, first_tile, n_slots);
}
#endif

#if B200PT_NSPEC == 3  // spectrum-independent: compiled once, in the RGBSpectrum translation unit
// ----------------------------------------------------------------------- trace
// Persistent warps; every lane owns one ray at a time.  A lane whose ray is
// finished parks until fewer than `refill_lanes` lanes of the warp are
// still traversing (TraceArgs::refill_lanes); then the warp reconverges, finished rays are written out
// (+ classified by BSDF family with warp-aggregated appends) and idle lanes
// fetch new rays -- so one long ray never keeps 31 lanes idle.
// Every traversal kernel takes the mask test as its class ALPHA: AlphaTest for scenes with alpha masks, NoAlpha
// (wbvh_traverse.cuh) for the rest; the launchers pick it from TraceArgs::alpha_masks.

// Alpha masks inside intersection (Triangle::Intersect / IntersectP, shapes/triangle.cpp:332-337, 531-570): a candidate
// the watertight test accepted is rejected when a mask of its mesh evaluates to exactly 0 at uvHit = b0 uv0 + b1 uv1 +
// b2 uv2 (GetUVs' defaults (0,0) (1,0) (1,1) without mesh uvs).  That SurfaceInteraction has no differentials, so
// UVMapping2D::Map gives zero footprints and both MIPMap::Lookup overloads reduce to triangle(0, st).  Closest hits test
// alpha only; any-hit rays (IntersectP) test alpha, then shadowalpha, unless the launch answers volpath's shadow rays,
// whose Tr intersects with Intersect.  IntersectP also rejects a masked triangle whose geometric normal is zero: such
// triangles never enter a tree (B200PT_TRI_DEGENERATE).  Shape::Pdf / Sample ignore masks, and so do the re-intersections
// of an accepted hit (hit_distance, fill_isect) and the light-pdf test of estimate_direct: they call triangle_test alone.
struct AlphaTest {
    static constexpr bool enabled = true;
    const DevAlphaMask *masks;
    const int32_t *ids;  // TraceArgs::alpha_ids
    const F4 *tri_uv;    // at the first triangle of the tree being walked
    int any_shadow;
    B200_HD static AlphaTest of(const TraceArgs &a) {
        AlphaTest t;
        t.masks = a.alpha_masks;
        t.ids = a.alpha_ids;
        t.tri_uv = a.tri_uv;
        t.any_shadow = a.alpha_any_shadow;
        return t;
    }
    // the same masks for the tree whose triangles start at tri_off in the scene's arrays (an object's tree)
    B200_HD AlphaTest at(uint32_t tri_off) const {
        AlphaTest t = *this;
        if (t.tri_uv) t.tri_uv += (size_t)tri_off * 2;
        return t;
    }
    // ImageTexture<Float, Float>::Evaluate (imagemap.h:83-92) or ConstantTexture(0) == 0
    B200_HD bool zero(int m, float u, float v) const {
        const DevAlphaMask &M = masks[m];
        if (M.mip.levels == 0) return true;
        return mip_triangle(M.mip, 0, M.su * u + M.du, M.sv * v + M.dv).c[0] == 0.f;
    }
    B200_HD bool rejects(bool any_hit, uint32_t ti, uint32_t prim, uint32_t mflags, const TriHit &h) const {
        float uv[6] = {0.f, 0.f, 1.f, 0.f, 1.f, 1.f};
        if (mflags & B200PT_TRI_HAS_UVS) {
            const F4 a = ld_f4(tri_uv + (size_t)ti * 2), b = ld_f4(tri_uv + (size_t)ti * 2 + 1);
            uv[0] = a.x;
            uv[1] = a.y;
            uv[2] = a.z;
            uv[3] = a.w;
            uv[4] = b.x;
            uv[5] = b.y;
        }
        const float u = h.b0 * uv[0] + h.b1 * uv[2] + h.b2 * uv[4];
        const float v = h.b0 * uv[1] + h.b1 * uv[3] + h.b2 * uv[5];
        const int alpha = ids[(size_t)prim * 2];
        if (alpha >= 0 && zero(alpha, u, v)) return true;
        if (any_hit && any_shadow) {
            const int shadow = ids[(size_t)prim * 2 + 1];
            if (shadow >= 0 && zero(shadow, u, v)) return true;
        }
        return false;
    }
};

__device__ __forceinline__ TravBounds instance_bounds(const DevInstance &in) {
    TravBounds b;
    for (int a = 0; a < 3; ++a) {
        b.lo[a] = in.obj_lo[a];
        b.hi[a] = in.obj_hi[a];
    }
    b.scale = in.obj_scale;
    return b;
}

#ifdef B200PT_HOST_EMU
// CPU check build: the warp-synchronous kernel below cannot run one lane at a time; every ray takes the per-ray
// routine the kernel's lanes step through (traverse_wbvh = trav_step until done) and retires like a lane does.
template <bool ANY_HIT, bool CLASSIFY, bool COUNT, class ALPHA>
void trace_walk(const TraceArgs a, const ALPHA alpha) {
    const uint32_t n = *a.count;
    TraceCounters ctr;
    ctr.nodes = ctr.tris = 0;
    uint32_t overflow = 0;
    uint32_t i;
    while (warp_fetch(a.work, n, &i)) {
        const uint32_t slot = a.queue ? a.queue[i] : i;
        const float4 o4 = a.ray_o[(size_t)slot * a.stride];
        const float4 d4 = a.ray_d[(size_t)slot * a.stride];
        TriHit hit;
        hit.t = hit.b0 = hit.b1 = hit.b2 = 0.f;
        const uint32_t best = traverse_wbvh<ANY_HIT, COUNT>(a.nodes, a.tri_base, a.tris, a.bounds, a.lut, v3(o4), v3(d4),
                                                            a.t_max_from_w ? o4.w : a.fixed_t_max, &hit, &ctr, &overflow, alpha);
        if (ANY_HIT) {
            slot_out(a.occ_out, slot, a.out_stride) = best != B200PT_MISS ? 1 : 0;
            continue;
        }
        if (a.hit_out) slot_out(a.hit_out, slot, a.out_stride) = best;
        if (a.full_out) {
            b200pt_hit r;
            r.triangle = best != B200PT_MISS ? (int32_t)__float_as_uint(ld_f4(a.tris + (size_t)best * 3).w) : -1;
            r.t = hit.t;
            r.b0 = hit.b0;
            r.b1 = hit.b1;
            a.full_out[slot] = r;
        }
        if (CLASSIFY && best != B200PT_MISS)
            append_family(a.q_mat, a.qcount_mat, hit_family(a.materials, __float_as_uint(ld_f4(a.tris + (size_t)best * 3 + 1).w)), slot);
    }
    if (COUNT) {
        atomicAdd(&a.stats[ANY_HIT ? 5 : 3], (unsigned long long)ctr.nodes);
        atomicAdd(&a.stats[ANY_HIT ? 6 : 4], (unsigned long long)ctr.tris);
    }
    if (overflow && a.stats) atomicAdd(&a.stats[7], (unsigned long long)overflow);
}
#else
// The ray as the triangle test sees it and the result so far (TravRay) live in shared memory, one column per
// thread (conflict-free): the node loop -- where a lane spends its time -- keeps only the box-test state in
// registers, the much rarer triangle phase fetches what it needs.
#define B200PT_RAY_WORDS 21  // 0-2 o, 3-5 shear, 6 kz, 7 tMax, 8 best, 9-12 hit, 13 t0, 14-16 1/d, 17-19 origin/d, 20 span floor
__device__ __forceinline__ void ray_store(float *col, const TravRay &R) {
    col[0 * 128] = R.o.x;
    col[1 * 128] = R.o.y;
    col[2 * 128] = R.o.z;
    col[3 * 128] = R.sh.Sx;
    col[4 * 128] = R.sh.Sy;
    col[5 * 128] = R.sh.Sz;
    col[6 * 128] = __int_as_float(R.sh.kz);
    col[7 * 128] = R.tmax;
    col[8 * 128] = __uint_as_float(R.best);
    col[9 * 128] = R.hit.t;
    col[10 * 128] = R.hit.b0;
    col[11 * 128] = R.hit.b1;
    col[12 * 128] = R.hit.b2;
    col[13 * 128] = R.t0;
    col[14 * 128] = R.iu[0];
    col[15 * 128] = R.iu[1];
    col[16 * 128] = R.iu[2];
    col[17 * 128] = R.ou[0];
    col[18 * 128] = R.ou[1];
    col[19 * 128] = R.ou[2];
    col[20 * 128] = R.span_floor;
}
// what trav_rescale reads (fetched only after a closest hit shortened the ray)
__device__ __forceinline__ void ray_load_scale(const float *col, TravRay &R) {
    R.t0 = col[13 * 128];
    R.iu[0] = col[14 * 128];
    R.iu[1] = col[15 * 128];
    R.iu[2] = col[16 * 128];
    R.ou[0] = col[17 * 128];
    R.ou[1] = col[18 * 128];
    R.ou[2] = col[19 * 128];
    R.span_floor = col[20 * 128];
}
__device__ __forceinline__ void ray_load(const float *col, TravRay &R) {
    R.o = mk(col[0 * 128], col[1 * 128], col[2 * 128]);
    R.sh.Sx = col[3 * 128];
    R.sh.Sy = col[4 * 128];
    R.sh.Sz = col[5 * 128];
    R.sh.kz = __float_as_int(col[6 * 128]);
    R.sh.kx = R.sh.kz == 2 ? 0 : R.sh.kz + 1;
    R.sh.ky = R.sh.kx == 2 ? 0 : R.sh.kx + 1;
    R.tmax = col[7 * 128];
    R.best = __float_as_uint(col[8 * 128]);
    R.hit.t = R.hit.b0 = R.hit.b1 = R.hit.b2 = 0.f;  // outputs of the triangle phase (stored again only after a hit)
}
__device__ __forceinline__ void ray_store_hit(float *col, const TravRay &R) {
    col[7 * 128] = R.tmax;
    col[8 * 128] = __uint_as_float(R.best);
    col[9 * 128] = R.hit.t;
    col[10 * 128] = R.hit.b0;
    col[11 * 128] = R.hit.b1;
    col[12 * 128] = R.hit.b2;
}

// Writes out the lane's ray if it is finished (`fin`; its record is the column my_ray, its stack state sp) and, with
// CLASSIFY, appends its slot to the queue of the hit's BSDF family.  hit_inst (k_trace2): where the instance of a hit
// goes (record word 21), or nullptr.  Every lane of the warp must call it (converged).
template <bool ANY_HIT, bool CLASSIFY>
__device__ __forceinline__ void retire_ray(const TraceArgs &a, const float *my_ray, bool fin, uint32_t slot, uint32_t sp,
                                           uint32_t *hit_inst) {
    int family = -1;
    if (fin) {
        const uint32_t best = __float_as_uint(my_ray[8 * 128]);
        if (ANY_HIT) {
            slot_out(a.occ_out, slot, a.out_stride) = best != B200PT_MISS ? 1 : 0;
        } else {
            if (a.hit_out) slot_out(a.hit_out, slot, a.out_stride) = best;
            if (hit_inst && best != B200PT_MISS) slot_out(hit_inst, slot, a.out_stride) = __float_as_uint(my_ray[21 * 128]);
            if (a.full_out) {
                b200pt_hit r;
                r.triangle = best != B200PT_MISS ? (int32_t)__float_as_uint(ld_f4(a.tris + (size_t)best * 3).w) : -1;
                r.t = my_ray[9 * 128];
                r.b0 = my_ray[10 * 128];
                r.b1 = my_ray[11 * 128];
                a.full_out[slot] = r;
            }
            if (CLASSIFY && best != B200PT_MISS)
                family = hit_family(a.materials, __float_as_uint(ld_f4(a.tris + (size_t)best * 3 + 1).w));
        }
        if ((sp & B200PT_SP_OVERFLOW) && a.stats) atomicAdd(&a.stats[7], 1ull);
    }
    if (CLASSIFY) append_family(a.q_mat, a.qcount_mat, family, slot);
}

template <bool ANY_HIT, bool CLASSIFY, bool COUNT, class ALPHA>
__device__ __forceinline__ void trace_walk(const TraceArgs a, const ALPHA alpha) {
    // the slot-permutation table of the node test (wbvh_traverse.cuh), one copy per CTA
    __shared__ __align__(16) uint8_t s_lut[B200PT_LUT_BYTES];
    __shared__ float s_ray[B200PT_RAY_WORDS * 128];
    reinterpret_cast<uint4 *>(s_lut)[threadIdx.x] = __ldg(reinterpret_cast<const uint4 *>(a.lut) + threadIdx.x);
    __syncthreads();
    float *const my_ray = s_ray + threadIdx.x;
    const uint32_t n = *a.count;
    TraceCounters ctr;
    ctr.nodes = ctr.tris = 0;
    Trav T;
    TravStack S;
    uint32_t slot = 0, pend_x = 0, pend_y = 0;
    bool has = false, fin = false, exhausted = false;
    while (true) {
        // ---- converged: retire finished rays
        retire_ray<ANY_HIT, CLASSIFY>(a, my_ray, fin, slot, T.sp, nullptr);
        fin = false;
        // ---- converged: idle lanes fetch new rays.  warp_append written out: through warp_append this kernel
        // compiles to another schedule, and cfg4 took 8042 and 8044 ms per step against 8030 and 8030 written out
        // (bench.py, the two builds alternating, H100 80GB HBM3 at 700 W)
        {
            const bool want = !has && !exhausted;
            const uint32_t mask = __ballot_sync(FULL_MASK, want);
            if (mask) {
                const int lane = threadIdx.x & 31;
                const int leader = __ffs(mask) - 1;
                uint32_t base = 0;
                if (lane == leader) base = atomicAdd(a.work, (uint32_t)__popc(mask));
                base = __shfl_sync(FULL_MASK, base, leader);
                if (want) {
                    const uint32_t i = base + (uint32_t)__popc(mask & ((1u << lane) - 1u));
                    if (i < n) {
                        slot = a.queue ? a.queue[i] : i;
                        const float4 o4 = a.ray_o[(size_t)slot * a.stride];
                        const float4 d4 = a.ray_d[(size_t)slot * a.stride];
                        TravRay R;
                        trav_init(T, R, v3(o4), v3(d4), a.t_max_from_w ? o4.w : a.fixed_t_max, a.bounds);
                        ray_store(my_ray, R);
                        pend_y = 0;
                        has = true;
                    } else {
                        exhausted = true;
                    }
                }
            }
        }
        if (__ballot_sync(FULL_MASK, has) == 0) break;
        // ---- traverse until this lane's ray is done or the warp is mostly idle.
        // Leaf triangles are not intersected the moment a node step finds them: the watertight test is
        // long and typically only two or three lanes have triangles after a given step.  Each lane
        // parks its triangle group in (pend_x, pend_y); the lanes converged here run the triangle phase
        // together once enough of them have work (a.postpone_pct % of the converged lanes), or when a
        // lane needs it now (it found a second group, or has nothing else left to do).
        while (has) {
            uint32_t ng_x = 0, ng_y = 0;
            const bool node_work = (T.cur_y & 0xff000000u) != 0;
            if (node_work)
                trav_node_phase<!ANY_HIT, COUNT>(T, S, a.nodes, a.tri_base, s_lut, &ng_x, &ng_y, &ctr);
            bool must = false;
            if (ng_y) {
                if (pend_y) {
                    must = true;  // no room: flush the parked group now, park the new one after
                } else {
                    pend_x = ng_x;
                    pend_y = ng_y;
                    ng_y = 0;
                }
            }
            const bool out_of_nodes = (T.cur_y & 0xff000000u) == 0 && (T.sp & B200PT_SP_MASK) == 0;
            // one warp reduction instead of three votes: byte 0 counts parked lanes, byte 1 urgent, byte 2 starving
            const unsigned act = __activemask();
            const bool starving_me = out_of_nodes && pend_y != 0;
            const unsigned counts = __reduce_add_sync(
                act, (pend_y != 0 ? 1u : 0u) | ((must || (starving_me && a.postpone_pct <= 0)) ? 0x100u : 0u) |
                         (starving_me ? 0x10000u : 0u));
            const int n_act = __popc(act), n_parked = (int)(counts & 0xffu), n_starving = (int)((counts >> 16) & 0xffu);
            // run the triangle phase if someone must, if enough lanes parked work, or if so many lanes are
            // only waiting for it that the node phase itself would run half empty
            if ((counts & 0xff00u) || n_parked * 100 >= n_act * a.postpone_pct || n_starving * 4 >= n_act) {
                bool done = false;
                if (pend_y) {
                    TravRay R;
                    ray_load(my_ray, R);
                    const uint32_t before = R.best;
                    done = trav_tri_phase<ANY_HIT, COUNT>(R, a.tri_base, a.tris, pend_x, pend_y, &ctr, alpha);
                    if (R.best != before) {
                        ray_store_hit(my_ray, R);
                        if (!ANY_HIT) {  // the ray got shorter: the box parameter ends at the hit from now on
                            ray_load_scale(my_ray, R);
                            trav_rescale(T, R, R.tmax);
                        }
                    }
                }
                pend_x = ng_x;
                pend_y = ng_y;
                if (done) {
                    has = false;
                    fin = true;
                    pend_y = 0;
                }
            }
            if (has && !trav_next_group(T, S) && pend_y == 0) {
                has = false;
                fin = true;
            }
            if (__popc(__activemask()) < a.refill_lanes) break;
        }
        __syncwarp();
    }
    if (COUNT) {
        atomicAdd(&a.stats[ANY_HIT ? 5 : 3], (unsigned long long)ctr.nodes);
        atomicAdd(&a.stats[ANY_HIT ? 6 : 4], (unsigned long long)ctr.tris);
    }
}

// ---------------------------------------------------------------- two-level traversal (scenes with object instances)
// TransformedPrimitive::Intersect / IntersectP (core/primitive.cpp:70-106) inside the persistent kernel: a lane walks
// the top-level tree (triangles outside objects), then the tree over the instances' leaf boxes; a leaf of that tree
// names instances, and each candidate that passes its leaf-box gate takes the lane -- with the ray transformed into the
// object's space -- through that object's own tree, after which the walk over the instances resumes.  One set of
// box-test constants lives in registers (re-derived when the lane changes space: once per instance entered, not per
// node); what the lane must come back to waits on the same traversal stack behind a marked entry.  Replaces the
// one-batch-of-32-rays walk of k_spheres for the instances.
#define B200PT_RAY_WORDS2 24  // k_trace's record + 21 instance of the hit, 22 world tMax, 23 current instance
#define B200PT_MARK 0x80000000u  // stack entry x: "what follows is what the lane left behind when it entered an instance"
template <bool ANY_HIT, bool CLASSIFY, class ALPHA>
__global__ void __launch_bounds__(128, 6) k_trace2(const TraceArgs a) {
    __shared__ __align__(16) uint8_t s_lut[B200PT_LUT_BYTES];
    __shared__ float s_ray[B200PT_RAY_WORDS2 * 128];
    reinterpret_cast<uint4 *>(s_lut)[threadIdx.x] = __ldg(reinterpret_cast<const uint4 *>(a.lut) + threadIdx.x);
    __syncthreads();
    float *const my_ray = s_ray + threadIdx.x;
    const uint32_t n = *a.count;
    TraceCounters ctr;
    ctr.nodes = ctr.tris = 0;
    Trav T;
    TravStack S;
    uint32_t slot = 0, pend_x = 0, pend_y = 0;
    uint32_t noff = 0, toff = 0;  // the tree the lane is in: offsets of its nodes / triangles inside the scene's arrays
    int phase = 0;                // 0: top-level tree, 1: tree over the instances, 2: inside an instance
    bool has = false, fin = false, exhausted = false;
    bool want_exit = false;       // the object's tree is exhausted: the lane waits to go back to the world ray
    // (re)derives the box-test constants and the triangle-test record for a ray in the space the lane enters;
    // the position on the stack and the result so far are the lane's own and stay
    auto enter_space = [&](const V3 &o, const V3 &d, float tmax, const TravBounds &B) {
        TravRay R;
        const int sp = T.sp;
        trav_init(T, R, o, d, tmax, B);
        T.sp = sp;
        my_ray[0 * 128] = R.o.x;
        my_ray[1 * 128] = R.o.y;
        my_ray[2 * 128] = R.o.z;
        my_ray[3 * 128] = R.sh.Sx;
        my_ray[4 * 128] = R.sh.Sy;
        my_ray[5 * 128] = R.sh.Sz;
        my_ray[6 * 128] = __int_as_float(R.sh.kz);
        my_ray[7 * 128] = R.tmax;
        my_ray[13 * 128] = R.t0;
        my_ray[14 * 128] = R.iu[0];
        my_ray[15 * 128] = R.iu[1];
        my_ray[16 * 128] = R.iu[2];
        my_ray[17 * 128] = R.ou[0];
        my_ray[18 * 128] = R.ou[1];
        my_ray[19 * 128] = R.ou[2];
        my_ray[20 * 128] = R.span_floor;
    };
    auto world_ray = [&](V3 *o, V3 *d) {
        const float4 o4 = a.ray_o[(size_t)slot * a.stride];
        const float4 d4 = a.ray_d[(size_t)slot * a.stride];
        *o = v3(o4);
        *d = v3(d4);
    };
    while (true) {
        // ---- converged: retire finished rays
        retire_ray<ANY_HIT, CLASSIFY>(a, my_ray, fin, slot, T.sp, a.hit_inst_out);
        fin = false;
        // ---- converged: idle lanes fetch new rays
        {
            const bool want = !has && !exhausted;
            const uint32_t i = warp_append(a.work, want);
            if (want) {
                if (i < n) {
                    slot = a.queue ? a.queue[i] : i;
                    const float4 o4 = a.ray_o[(size_t)slot * a.stride];
                    const float4 d4 = a.ray_d[(size_t)slot * a.stride];
                    const float tmax = a.t_max_from_w ? o4.w : a.fixed_t_max;
                    T.sp = 0;
                    phase = 0;
                    want_exit = false;
                    noff = toff = 0;
                    enter_space(v3(o4), v3(d4), tmax, a.bounds);
                    my_ray[8 * 128] = __uint_as_float(B200PT_MISS);
                    my_ray[9 * 128] = my_ray[10 * 128] = my_ray[11 * 128] = my_ray[12 * 128] = 0.f;
                    my_ray[21 * 128] = __uint_as_float(0u);
                    my_ray[22 * 128] = tmax;  // the world ray's tMax
                    pend_y = 0;
                    has = true;
                } else {
                    exhausted = true;
                }
            }
        }
        if (__ballot_sync(FULL_MASK, has) == 0) break;
        while (has) {
            uint32_t ng_x = 0, ng_y = 0;
            // Entering an instance leaves ONE group of untried candidates behind, so in the tree over the instances a lane
            // holds (takes no node step) while it has a leaf group; a lane that is done with an object's tree waits the
            // same way.  Both wait for company: changing space is ~900 instructions and runs once the usual share of the
            // warp's lanes has something parked (triangles, candidates, a way back), not one lane at a time.
            const bool hold = (phase == 1 && pend_y != 0) || want_exit;
            const bool node_work = !hold && (T.cur_y & 0xff000000u) != 0;
            if (node_work)
                trav_node_phase<!ANY_HIT, false>(T, S, a.nodes + (size_t)noff * 4, a.tri_base + noff, s_lut, &ng_x, &ng_y, &ctr);
            bool must = false;
            if (ng_y) {
                if (pend_y) {
                    must = true;  // two groups: flush the parked one now, park the new one after
                } else {
                    pend_x = ng_x;
                    pend_y = ng_y;
                    ng_y = 0;
                }
            }
            const bool out_of_nodes = (T.cur_y & 0xff000000u) == 0;  // (what is left on the stack waits behind the parked group)
            const unsigned act = __activemask();
            const bool parked_me = pend_y != 0 || want_exit;
            const bool idle_me = hold || (phase == 1 && pend_y != 0) || (out_of_nodes && pend_y != 0);
            const unsigned counts = __reduce_add_sync(
                act, (parked_me ? 1u : 0u) | ((must || (idle_me && a.postpone_pct <= 0)) ? 0x100u : 0u) | (idle_me ? 0x10000u : 0u));
            const int n_act = __popc(act), n_parked = (int)(counts & 0xffu), n_idle = (int)((counts >> 16) & 0xffu);
            if ((counts & 0xff00u) || n_parked * 100 >= n_act * a.postpone_pct || n_idle * 4 >= n_act) {
                bool done = false;
                if (want_exit) {
                    // the object's tree is done: back to the world ray (its tMax is the hit's, if there was one) and to
                    // the walk over the instances -- first the candidates of the same leaf that were not tried
                    want_exit = false;
                    uint32_t ex, ey, gx, gy;
                    T.sp -= 2;
                    S.pop((T.sp & B200PT_SP_MASK) + 1, &ex, &ey);
                    S.pop(T.sp & B200PT_SP_MASK, &gx, &gy);
                    V3 ro, rd;
                    world_ray(&ro, &rd);
                    noff = a.tlas_node_off;
                    toff = a.tlas_tri_off;
                    phase = 1;
                    enter_space(ro, rd, my_ray[22 * 128], a.tlas_bounds);
                    T.cur_x = gx;
                    T.cur_y = gy;
                    if (ey) {
                        pend_x = ex;  // marked: already a triangle group
                        pend_y = ey;
                    }
                } else if (pend_y && phase == 1) {
                    // leaf of the tree over the instances: its "triangles" name instances; the first candidate whose
                    // leaf box the ray (with its current tMax) enters takes the lane into that object's tree
                    uint32_t tg_x, tg_y;
                    if (pend_x & B200PT_MARK) {  // candidates left over from before an instance was entered: already triangles
                        tg_x = pend_x & ~B200PT_MARK;
                        tg_y = pend_y;
                    } else {
                        leaf_group_triangles(a.tri_base + noff, pend_x, pend_y, &tg_x, &tg_y);
                    }
                    pend_y = 0;
                    V3 ro, rd;
                    world_ray(&ro, &rd);
                    const float wtmax = my_ray[22 * 128];
                    while (tg_y) {
                        const int j = msb32(tg_y);
                        tg_y &= ~(1u << j);
                        const uint32_t k = __float_as_uint(ld_f4(a.tris + (size_t)(toff + tg_x + (uint32_t)j) * 3).w);  // TriRecord::prim
                        const DevInstance &in = a.instances[k];
                        if (!instance_leaf_test(in, ro, rd, wtmax)) continue;
                        // left behind: the group being walked and the candidates not tried yet
                        if ((T.sp & B200PT_SP_MASK) + 2 > B200PT_STACK) {
                            T.sp |= B200PT_SP_OVERFLOW;
                            break;
                        }
                        S.push(T.sp & B200PT_SP_MASK, T.cur_x, T.cur_y);
                        S.push((T.sp & B200PT_SP_MASK) + 1, tg_x | B200PT_MARK, tg_y);
                        T.sp += 2;
                        V3 o2, d2;
                        float tm2;
                        instance_ray(in, ro, rd, wtmax, &o2, &d2, &tm2);
                        enter_space(o2, d2, tm2, instance_bounds(in));
                        noff = in.node_off;
                        toff = in.tri_off;
                        my_ray[23 * 128] = __uint_as_float(k);
                        phase = 2;
                        break;
                    }
                } else if (pend_y) {
                    TravRay R;
                    ray_load(my_ray, R);
                    R.best = B200PT_MISS;  // (an index inside this tree; the record keeps scene-wide ones)
                    done = trav_tri_phase<ANY_HIT, false>(R, a.tri_base + noff, a.tris + (size_t)toff * 3, pend_x, pend_y, &ctr, ALPHA::of(a).at(toff));
                    if (R.best != B200PT_MISS) {
                        R.best += toff;
                        ray_store_hit(my_ray, R);
                        if (!ANY_HIT) {
                            ray_load_scale(my_ray, R);
                            trav_rescale(T, R, R.tmax);
                        }
                        if (phase == 2) my_ray[21 * 128] = my_ray[23 * 128];  // the instance of the hit
                        my_ray[22 * 128] = R.tmax;                            // r.tMax = ray.tMax (primitive.cpp:91 / :120)
                    }
                    pend_y = 0;
                }
                if (ng_y) {  // the second group found in this step (only outside the tree over the instances)
                    pend_x = ng_x;
                    pend_y = ng_y;
                }
                if (done) {
                    has = false;
                    fin = true;
                    pend_y = 0;
                }
            }
            // ---- the next group of the current tree, or (later, in company) back out of an instance, or on to the next tree, or done
            if (has && !want_exit && (T.cur_y & 0xff000000u) == 0) {
                bool more = false, blocked = false;
                while (!more && !blocked) {
                    if ((T.sp & B200PT_SP_MASK) == 0) break;
                    uint32_t ex, ey;
                    S.pop((T.sp & B200PT_SP_MASK) - 1, &ex, &ey);
                    if (!(ex & B200PT_MARK)) {
                        --T.sp;
                        T.cur_x = ex;
                        T.cur_y = ey;
                        more = (ey & 0xff000000u) != 0;
                    } else {
                        blocked = true;  // an object's tree is exhausted: leave it once its parked triangles are tested
                        if (pend_y == 0) want_exit = true;
                    }
                }
                if (!more && !blocked && pend_y == 0) {
                    if (phase == 0 && a.n_instances > 0) {
                        // the top-level triangles are done: on to the instances, with the ray's tMax so far
                        V3 ro, rd;
                        world_ray(&ro, &rd);
                        noff = a.tlas_node_off;
                        toff = a.tlas_tri_off;
                        phase = 1;
                        enter_space(ro, rd, my_ray[22 * 128], a.tlas_bounds);
                        if ((T.cur_y & 0xff000000u) == 0) {
                            has = false;
                            fin = true;
                        }
                    } else {
                        has = false;
                        fin = true;
                    }
                }
            }
            if (__popc(__activemask()) < a.refill_lanes) break;
        }
        __syncwarp();
    }
}
#endif  // B200PT_HOST_EMU

template <bool ANY_HIT, bool CLASSIFY, bool COUNT, class ALPHA>
__global__ void __launch_bounds__(128, B200PT_TRACE_CTAS) k_trace(const TraceArgs a) {
    trace_walk<ANY_HIT, CLASSIFY, COUNT>(a, ALPHA::of(a));
}

// ---------------------------------------------------------------------- instances
// All instances against one ray, as a resumable state machine: through the tree over their leaf boxes when there is
// one (its leaf "triangles" carry instance numbers), else one by one.  Each lane walks the tree over the instances'
// boxes, picks the next candidate instance, or takes ONE step inside that instance's tree per call of step(), so that
// the lanes of a warp meet again after every step instead of after whole nested traversals (measured with nested loops:
// 2.4 of 32 lanes active per instruction) and a lane whose ray is done can take the next ray (k_spheres).
template <bool ANY_HIT, class ALPHA>
struct InstanceWalk {
    Trav T1, T2;
    TravRay R1, R2;
    TravStack S1, S2;
    V3 ro, rd;
    uint32_t pend_x, pend_y, cur_inst, cur_tri_off, overflow;
    const U4 *bn;
    const uint32_t *bb;
    const F4 *bt;
    int state;  // 0: instance tree, 1: next candidate, 2: inside an instance, 3: done
    uint32_t next_linear;  // scenes without a tree over the instances: the next instance to try
    // results
    uint32_t best, inst;
    TriHit hit;

    __device__ void init(const TraceArgs &a, const V3 &o, const V3 &d, float tmax) {
        ro = o;
        rd = d;
        best = B200PT_MISS;
        inst = 0;
        hit.t = hit.b0 = hit.b1 = hit.b2 = 0.f;
        pend_x = pend_y = cur_inst = cur_tri_off = overflow = 0;
        next_linear = 0;
        bn = nullptr;
        bb = nullptr;
        bt = nullptr;
        state = 0;
        trav_init(T1, R1, o, d, tmax, a.tlas_bounds);
        if (a.tlas_node_off == 0u) {  // no tree: T1 only carries the ray's tMax
            T1.cur_y = 0u;
            R1.tmax = tmax;
            state = 1;
        }
        T2 = T1;
        R2 = R1;
        T2.cur_y = 0u;
    }
    __device__ float tmax() const { return R1.tmax; }
    __device__ bool enter(const TraceArgs &a, uint32_t k) {
        const DevInstance &in = a.instances[k];
        if (!instance_leaf_test(in, ro, rd, R1.tmax)) return false;
        V3 o2, d2;
        float tm2;
        instance_ray(in, ro, rd, R1.tmax, &o2, &d2, &tm2);
        trav_init(T2, R2, o2, d2, tm2, instance_bounds(in));
        bn = a.nodes + (size_t)in.node_off * 4;
        bb = a.tri_base + in.node_off;
        bt = a.tris + (size_t)in.tri_off * 3;
        cur_inst = k;
        cur_tri_off = in.tri_off;
        return true;
    }
    // one step; true when the walk is complete
    __device__ bool step(const TraceArgs &a) {
        TraceCounters ctr;
        if (state == 2) {
            if (!(T2.cur_y & 0xff000000u) || trav_step<ANY_HIT, false>(T2, R2, S2, bn, bb, bt, a.lut, &ctr, ALPHA::of(a).at(cur_tri_off))) {
                overflow += (T2.sp & B200PT_SP_OVERFLOW) ? 1u : 0u;
                T2.sp &= B200PT_SP_MASK;
                state = 1;
                if (R2.best != B200PT_MISS) {
                    best = cur_tri_off + R2.best;
                    inst = cur_inst;
                    hit = R2.hit;
                    R1.tmax = R2.hit.t;  // r.tMax = ray.tMax (primitive.cpp:91)
                    trav_rescale(T1, R1, R1.tmax);
                    if (ANY_HIT) state = 3;
                }
            }
        } else if (state == 1) {
            if (a.tlas_node_off == 0u) {
                if (next_linear < a.n_instances) {
                    if (enter(a, next_linear)) state = 2;
                    ++next_linear;
                } else {
                    state = 3;
                }
            } else if (pend_y) {
                const int j = msb32(pend_y);
                pend_y &= ~(1u << j);
                const F4 *tt = a.tris + (size_t)a.tlas_tri_off * 3;
                const uint32_t k = __float_as_uint(ld_f4(tt + (size_t)(pend_x + (uint32_t)j) * 3).w);  // TriRecord::prim
                if (enter(a, k)) state = 2;
            } else {
                state = 0;
            }
        } else if (state == 0) {
            const U4 *tn = a.nodes + (size_t)a.tlas_node_off * 4;
            const uint32_t *tb1 = a.tri_base + a.tlas_node_off;
            if (T1.cur_y & 0xff000000u) {
                uint32_t lg_x = 0, lg_y = 0;
                trav_node_phase<!ANY_HIT, false>(T1, S1, tn, tb1, a.lut, &lg_x, &lg_y, &ctr);
                leaf_group_triangles(tb1, lg_x, lg_y, &pend_x, &pend_y);
                state = 1;
            } else if (!trav_next_group(T1, S1)) {
                state = 3;
            }
        }
        if (state == 3) {
            overflow += (T1.sp & B200PT_SP_OVERFLOW) ? 1u : 0u;
            T1.sp &= B200PT_SP_MASK;
            if (overflow && a.stats) atomicAdd(&a.stats[7], (unsigned long long)overflow);
            overflow = 0;
            return true;
        }
        return false;
    }
};

// ---------------------------------------------------------------------- spheres + instances
// Scene::Intersect / IntersectP for the Sphere shapes (not part of the BVH) and the object instances: the rays of
// the traversal launch that just finished (tMax shortened by its triangle hit).  Persistent warps; a lane that finished
// its ray takes the next one as soon as fewer than refill_lanes lanes of the warp are still walking (like k_trace).
template <bool ANY_HIT, bool CLASSIFY, class ALPHA>
__global__ void __launch_bounds__(128) k_spheres(const TraceArgs a) {
    const uint32_t n = *a.count;
#ifndef B200PT_HOST_EMU
    const int lane = threadIdx.x & 31;
#endif
    InstanceWalk<ANY_HIT, ALPHA> W;
    uint32_t slot = 0, best = B200PT_MISS;
    bool has = false, fin = false, exhausted = false, occluded = false;
    while (true) {
        // ---- converged: retire finished rays
        {
            int family = -1;
            if (fin) {
                if (ANY_HIT) {
                    if (occluded || W.best != B200PT_MISS) slot_out(a.occ_out, slot, a.out_stride) = 1;
                } else {
                    if (W.best != B200PT_MISS) {
                        best = W.best;
                        if (a.hit_out) slot_out(a.hit_out, slot, a.out_stride) = best;
                        if (a.hit_inst_out) slot_out(a.hit_inst_out, slot, a.out_stride) = W.inst;
                        if (a.full_out) {
                            b200pt_hit r;
                            r.triangle = (int32_t)__float_as_uint(ld_f4(a.tris + (size_t)best * 3).w);
                            r.t = W.hit.t;
                            r.b0 = W.hit.b0;
                            r.b1 = W.hit.b1;
                            a.full_out[slot] = r;
                        }
                    }
                    if (CLASSIFY && best != B200PT_MISS) {
                        const uint32_t mf = is_sphere_hit(best) ? a.spheres[best & SPHERE_HIT_MASK].mat_flags
                                                                : __float_as_uint(ld_f4(a.tris + (size_t)best * 3 + 1).w);
                        family = hit_family(a.materials, mf);
                    }
                }
            }
            if (CLASSIFY) append_family(a.q_mat, a.qcount_mat, family, slot);
            fin = false;
        }
        // ---- converged: idle lanes fetch new rays, test the spheres, set up the walk over the instances.  warp_append
        // written out (the check build's one-lane form below): through warp_append this kernel compiles to another
        // schedule, and cfg5rgb's separate pass (B200PT_NO_TRACE2=1) took 1762 and 1762 ms per step against 1748 and
        // 1748 written out (bench.py, the two builds alternating, H100 80GB HBM3 at 700 W)
        {
            const bool want = !has && !exhausted;
            uint32_t i = 0;
            bool got = false;
#ifdef B200PT_HOST_EMU
            if (want) {
                i = atomicAdd(a.sphere_work, 1u);
                got = i < n;
                exhausted = !got;
            }
#else
            const uint32_t mask = __ballot_sync(FULL_MASK, want);
            if (mask) {
                const int leader = __ffs(mask) - 1;
                uint32_t base = 0;
                if (lane == leader) base = atomicAdd(a.sphere_work, (uint32_t)__popc(mask));
                base = __shfl_sync(FULL_MASK, base, leader);
                if (want) {
                    i = base + (uint32_t)__popc(mask & ((1u << lane) - 1u));
                    got = i < n;
                    exhausted = !got;
                }
            }
#endif
            if (got) {
                slot = a.queue ? a.queue[i] : i;
                const float4 o4 = a.ray_o[(size_t)slot * a.stride];
                const float4 d4 = a.ray_d[(size_t)slot * a.stride];
                const V3 ro = v3(o4), rd = v3(d4);
                float tmax = a.t_max_from_w ? o4.w : a.fixed_t_max;
                best = B200PT_MISS;
                occluded = false;
                if (ANY_HIT) {
                    occluded = slot_out(a.occ_out, slot, a.out_stride) != 0;
                    for (uint32_t k = 0; k < a.n_spheres && !occluded; ++k) {
                        float t;
                        if (sphere_leaf_test(a.spheres[k], ro, rd, tmax) && sphere_intersect(a.spheres[k], ro, rd, tmax, &t, nullptr)) {
                            slot_out(a.occ_out, slot, a.out_stride) = 1;
                            occluded = true;
                        }
                    }
                } else {
                    if (a.hit_out) {
                        best = slot_out(a.hit_out, slot, a.out_stride);
                        if (best != B200PT_MISS) {  // ray.tMax after the triangle hit: Triangle::Intersect's t
                            const F4 *tp = a.tris + (size_t)best * 3;
                            const F4 t0 = ld_f4(tp), t1 = ld_f4(tp + 1), t2 = ld_f4(tp + 2);
                            V3 o2 = ro, d2 = rd;
                            if ((__float_as_uint(t1.w) & B200PT_TRI_INSTANCED) && a.hit_inst_out) {
                                // a triangle of an instanced object (found by the two-level kernel): the same ray parameter in
                                // the object's space (primitive.cpp:91)
                                float tm2;
                                instance_ray(a.instances[slot_out(a.hit_inst_out, slot, a.out_stride)], ro, rd, pt_inf(), &o2, &d2, &tm2);
                            }
                            TriHit h;
                            if (triangle_test(v3(t0), v3(t1), v3(t2), o2, make_shear(d2), pt_inf(), &h)) tmax = h.t;
                        }
                    } else if (a.full_out[slot].triangle >= 0) {
                        tmax = a.full_out[slot].t;
                        best = 0u;  // some top-level triangle (only its presence matters below: full_out keeps the record)
                    }
                    uint32_t sph = B200PT_MISS;
                    for (uint32_t k = 0; k < a.n_spheres; ++k) {
                        float t;
                        if (sphere_leaf_test(a.spheres[k], ro, rd, tmax) && sphere_intersect(a.spheres[k], ro, rd, tmax, &t, nullptr)) {
                            tmax = t;
                            sph = k;
                        }
                    }
                    if (sph != B200PT_MISS) {
                        best = SPHERE_HIT_BASE | sph;
                        if (a.hit_out) slot_out(a.hit_out, slot, a.out_stride) = best;
                        if (a.full_out) {
                            b200pt_hit r;
                            r.triangle = (int32_t)(a.n_tris + sph);
                            r.t = tmax;
                            r.b0 = r.b1 = 0.f;
                            a.full_out[slot] = r;
                        }
                    }
                }
                W.best = B200PT_MISS;
                if (a.n_instances && !(ANY_HIT && occluded)) {
                    W.init(a, ro, rd, tmax);
                    has = true;
                } else {
                    fin = true;  // nothing to walk: retire in the next round
                }
            }
        }
#ifdef B200PT_HOST_EMU
        while (has) {
            if (W.step(a)) {
                has = false;
                fin = true;
            }
        }
        if (!fin && exhausted) break;
#else
        if (__ballot_sync(FULL_MASK, has || fin) == 0) break;
        while (has) {
            if (W.step(a)) {
                has = false;
                fin = true;
            }
            if (__popc(__activemask()) < a.sphere_refill_lanes) break;
        }
        __syncwarp();
#endif
    }
}

#endif  // B200PT_NSPEC == 3
__device__ __forceinline__ DeltaLight delta_of(const DevLight &l, const Spec &intensity) {
    DeltaLight d;
    d.kind = l.kind;
    d.position = mk(l.position[0], l.position[1], l.position[2]);
    d.intensity = intensity;
    d.cos_total_width = l.cos_total_width;
    d.cos_falloff_start = l.cos_falloff_start;
    d.world_to_light = l.world_to_light;
    d.two_world_radius = l.two_world_radius;
    return d;
}

#if B200PT_NSPEC == 3
// ImageTexture::Evaluate (imagemap.h) through UVMapping2D::Map (texture.cpp:93-99)
__device__ __forceinline__ Spec texture_eval(const RenderDev *R, const DevTexBind &t, const TexGeom &g) {
    return mip_lookup(R->mipmaps[t.mip], t.su * g.u + t.du, t.sv * g.v + t.dv, t.su * g.dudx, t.sv * g.dvdx, t.su * g.dudy,
                      t.sv * g.dvdy);
}
// The material record of one hit: the material's textured parameters looked up, clamped and remapped like its
// ComputeScatteringFunctions does (matte.cpp:50-62, plastic.cpp:50-70, metal.cpp:64-80, glass.cpp:50-64, mirror.cpp:48-56);
// make_bsdf's black tests then decide the lobes per hit
__device__ void textured_material(const RenderDev *R, uint32_t mi, const TexGeom &g, b200pt_material *m) {
    const DevTexBind *tb = R->tex_bind + (size_t)mi * B200PT_TEX_SLOTS;
    float *const spectra[5] = {m->kd, m->ks, m->kt, m->eta, m->k};
    for (int slot = 0; slot < B200PT_TEX_SLOTS; ++slot) {
        const DevTexBind t = tb[slot];
        if (t.mip < 0) continue;
        const Spec v = texture_eval(R, t, g);
        if (slot <= B200PT_TEX_KT) {
            clamp_rgb(v, spectra[slot]);
        } else if (slot <= B200PT_TEX_K) {
            for (int c = 0; c < 3; ++c) spectra[slot][c] = v.c[c];
        } else {
            const float a = t.remap ? roughness_to_alpha(v.c[0]) : v.c[0];
            if (slot == B200PT_TEX_ROUGHNESS_U)
                m->alpha_x = a;
            else
                m->alpha_y = a;
        }
    }
}
#endif

// ----------------------------------------------------------------------- shade
struct DirectOut {
    uint32_t pend;
    V3 sh_o, sh_d, mi_o, mi_d;
    Spec A, B;
    // scenes with bounded media: the transmittance of the two rays is only known after they have walked through the
    // boundaries, so the factors stay apart: A = f, A2 = Li, wA = MIS weight (< 0: delta light, none), pdfA = lightPdf, and
    // the point the shadow ray is re-aimed at (p1 + error bounds + normal); B = f, wB = weight, pdfB = scatteringPdf
    Spec A2;
    float wA, pdfA, wB, pdfB;
    V3 p1, p1e, p1n;
};
// whether this translation unit carries the bounded-media code (the RGBSpectrum one)
#define B200PT_MEDIA_GENERAL (B200PT_NSPEC == 3)

// EstimateDirect (core/integrator.cpp:108-215), handleMedia = false,
// specular = false, for a DiffuseAreaLight on one triangle.  The two rays it
// needs are not traced here: the shadow ray and the BSDF-sampled ("MIS") ray
// are queued with the terms they gate (A and B).
// With R->has_medium (VolPathIntegrator, handleMedia = true, every ray inside one homogeneous medium) the two rays also
// carry a transmittance: an unoccluded shadow ray's is known here (VisibilityTester::Tr, light.cpp:63-81, every surface
// is opaque), and the MIS ray can only contribute if its closest hit is the light's own shape, whose distance Pdf_Li
// computes anyway (Scene::IntersectTr, scene.cpp:57-70).  `inMedium`: `is` is a MediumInteraction (p, wo; zero normal
// and error bounds) and the Henyey-Greenstein phase function takes the BSDF's place (integrator.cpp:131-137, :178-186).
template <bool VTX, int KINDS = KM_ALL>
__device__ void estimate_direct(const RenderDev *R, const Isect &is, const Bsdf &bsdf, const float uScattering[2],
                                int lightNum, const float uLight[2], DirectOut *out, bool inMedium = false, int med = 0) {
    // (VolPathIntegrator renders always run the general variant, so the lean one carries none of this)
    // `general`: media bounded by surfaces; `med` is the medium id around `is` and the rays' transmittance is left to
    // the walk kernels
    const bool general = B200PT_MEDIA_GENERAL && VTX && R->med_general != 0;
    const bool medium = VTX && R->has_medium != 0 && !general;
    const Spec sigmaT = medium ? medium_sigma_t(R) : rgb1(0.f);
    const float hgG = general ? (med >= 0 ? R->media_g[med] : 0.f) : R->med_g;
    if (!VTX) inMedium = false;
    out->A2 = rgb1(0.f);
    out->wA = out->pdfA = out->wB = out->pdfB = 0.f;
    out->p1 = out->p1e = out->p1n = mk(0.f, 0.f, 0.f);
    const DevLight &lightRef = R->lights[lightNum];
#if B200PT_NSPEC == 3
    if constexpr (VTX) {
        if (lightRef.kind == B200PT_LIGHT_INFINITE) {
            // an infinite light (PathIntegrator only: no medium): the shadow ray aims at ref.p + wi * 2 worldRadius like a
            // point light's, the MIS ray contributes Le(ray) if it hits nothing -- the light's record has tri == B200PT_MISS
            const DevInfinite &L = R->infinite[lightRef.two_sided];
            const int flagsNS = BSDF_ALL & ~BSDF_SPECULAR;
            out->pend = 0;
            out->sh_o = out->sh_d = out->mi_o = out->mi_d = mk(0.f, 0.f, 0.f);
            out->A = out->B = rgb1(0.f);
            V3 wi, pTarget;
            float lightPdf, scatteringPdf = 0.f;
            const Spec Li = infinite_sample_li(L, is.p, uLight, &wi, &lightPdf, &pTarget);
            if (lightPdf > 0 && !is_black(Li)) {
                const Spec f = bsdf_f<KINDS>(bsdf, is.wo, wi, flagsNS) * absdot(wi, bsdf.ns);
                scatteringPdf = bsdf_pdf<KINDS>(bsdf, is.wo, wi, flagsNS);
                if (!is_black(f)) {
                    const V3 origin = offset_ray_origin(is.p, is.pError, is.n, pTarget - is.p);
                    out->sh_o = origin;
                    out->sh_d = pTarget - origin;
                    const float weight = power_heuristic(lightPdf, scatteringPdf);
                    out->A = f * Li * weight / lightPdf;
                    out->pend |= PEND_LIGHT;
                }
            }
            int sampledType = 0;
            Spec f = bsdf_sample_f<KINDS>(bsdf, is.wo, &wi, uScattering, &scatteringPdf, flagsNS, &sampledType);
            f = f * absdot(wi, bsdf.ns);
            if (!is_black(f) && scatteringPdf > 0) {
                const float lpdf = infinite_pdf_li(L, wi);
                if (lpdf != 0) {  // `if (lightPdf == 0) return Ld;` (integrator.cpp:182): no MIS ray then
                    const float weight = power_heuristic(scatteringPdf, lpdf);
                    const Spec Le = infinite_le(L, wi);
                    out->B = is_black(Le) ? rgb1(0.f) : f * Le * weight / scatteringPdf;
                    out->mi_o = offset_ray_origin(is.p, is.pError, is.n, wi);
                    out->mi_d = wi;
                    out->pend |= PEND_BSDF;
                }
            }
            return;
        }
    }
#endif
    if (VTX && lightRef.kind != 0) {
        // delta light (scenes with delta lights always run the VTX variant): Sample_Li has pdf 1, there is no MIS weight
        // and no BSDF-sampling branch (integrator.cpp:147-148, :166)
        out->pend = 0;
        out->sh_o = out->sh_d = out->mi_o = out->mi_d = mk(0.f, 0.f, 0.f);
        out->A = out->B = rgb1(0.f);
        const DeltaLight dl = delta_of(lightRef, light_emit(R, lightNum, lightRef));
        V3 wiD, pTarget;
        const Spec LiD = delta_light_sample(dl, is.p, &wiD, &pTarget);
        if (!is_black(LiD)) {
            const Spec fD = inMedium ? rgb1(phase_hg(dot(is.wo, wiD), hgG))
                                     : bsdf_f<KINDS>(bsdf, is.wo, wiD, BSDF_ALL & ~BSDF_SPECULAR) * absdot(wiD, bsdf.ns);
            if (!is_black(fD)) {
                // SpawnRayTo(Interaction) towards a point without normal or error bounds (interaction.h:73-78)
                const V3 origin = offset_ray_origin(is.p, is.pError, is.n, pTarget - is.p);
                out->sh_o = origin;
                out->sh_d = pTarget - origin;
                const Spec LiT = medium ? LiD * medium_tr(sigmaT, out->sh_d, PT_SHADOW_TMAX) : LiD;  // Li *= Tr
                out->A = fD * LiT / 1.f;
                if (general) {
                    out->A = fD;
                    out->A2 = LiD;
                    out->wA = -1.f;
                    out->pdfA = 1.f;
                    out->p1 = pTarget;
                }
                out->pend |= PEND_LIGHT;
            }
        }
        return;
    }
    const DevLight light = lightRef;
    // a sphere light (scenes with spheres always run the VTX variant)
    const bool onSphere = VTX && is_sphere_hit(light.tri);
    const DevSphere *lsp = onSphere ? R->scene.spheres + (light.tri & SPHERE_HIT_MASK) : nullptr;
    const F4 *tp = R->scene.tris + (size_t)(onSphere ? 0u : light.tri) * 3;
    F4 t0 = {0.f, 0.f, 0.f, 0.f}, t1 = t0, t2 = t0;
    if (!onSphere) {
        t0 = ld_f4(tp);
        t1 = ld_f4(tp + 1);
        t2 = ld_f4(tp + 2);
    }
    const V3 p0 = v3(t0), p1 = v3(t1), p2 = v3(t2);
    const uint32_t lflags = __float_as_uint(t1.w);
    const bool lflip = (lflags & B200PT_TRI_FLIP) != 0, ldegenerate = (lflags & B200PT_TRI_DEGENERATE) != 0;
    TriShading lsh;
    load_shading<VTX>(R->scene, light.tri, lflags, &lsh);
    const Spec lemit = light_emit(R, lightNum, light);
    const int flagsNS = BSDF_ALL & ~BSDF_SPECULAR;
    out->pend = 0;
    out->sh_o = out->sh_d = out->mi_o = out->mi_d = mk(0.f, 0.f, 0.f);
    out->A = out->B = rgb1(0.f);
    V3 wi = mk(0.f, 0.f, 0.f);
    float lightPdf = 0.f, scatteringPdf = 0.f;
    // light.Sample_Li: diffuse.cpp:68-81, shape.cpp:56-70
    Spec Li = rgb1(0.f);
    LightSample ps;
    if (onSphere) {
        ps = sphere_sample(*lsp, is.p, is.pError, is.n, uLight, &lightPdf);  // already a solid-angle density
    } else {
        ps = triangle_sample(p0, p1, p2, lflip, lsh, uLight, &lightPdf);
        V3 w = ps.p - is.p;
        if (len2(w) == 0)
            lightPdf = 0;
        else {
            w = normalize(w);
            lightPdf *= len2(is.p - ps.p) / absdot(ps.n, -w);
            if (pt_isinf(lightPdf)) lightPdf = 0.f;
        }
    }
    if (lightPdf == 0 || len2(ps.p - is.p) == 0) {
        lightPdf = 0;
    } else {
        wi = normalize(ps.p - is.p);
        Li = (light.two_sided || dot(ps.n, -wi) > 0) ? lemit : rgb1(0.f);  // diffuse.h:56-58
    }
    if (lightPdf > 0 && !is_black(Li)) {
        Spec f;
        if (inMedium) {
            const float p = phase_hg(dot(is.wo, wi), hgG);
            f = rgb1(p);
            scatteringPdf = p;
        } else {
            f = bsdf_f<KINDS>(bsdf, is.wo, wi, flagsNS) * absdot(wi, bsdf.ns);
            scatteringPdf = bsdf_pdf<KINDS>(bsdf, is.wo, wi, flagsNS);
        }
        if (!is_black(f)) {
            // VisibilityTester::Unoccluded -> SpawnRayTo(Interaction), interaction.h:73-78
            const V3 origin = offset_ray_origin(is.p, is.pError, is.n, ps.p - is.p);
            const V3 target = offset_ray_origin(ps.p, ps.pError, ps.n, origin - ps.p);
            out->sh_o = origin;
            out->sh_d = target - origin;
            if (medium) Li = Li * medium_tr(sigmaT, out->sh_d, PT_SHADOW_TMAX);  // Li *= visibility.Tr(scene, sampler)
            const float weight = power_heuristic(lightPdf, scatteringPdf);
            out->A = f * Li * weight / lightPdf;
            if (general) {
                out->A = f;
                out->A2 = Li;
                out->wA = weight;
                out->pdfA = lightPdf;
                out->p1 = ps.p;
                out->p1e = ps.pError;
                out->p1n = ps.n;
            }
            out->pend |= PEND_LIGHT;
        }
    }
    // BSDF sampling with MIS (integrator.cpp:166-213)
    int sampledType = 0;
    Spec f;
    if (inMedium) {
        const float p = hg_sample_p(hgG, is.wo, &wi, uScattering);
        f = rgb1(p);
        scatteringPdf = p;
    } else {
        f = bsdf_sample_f<KINDS>(bsdf, is.wo, &wi, uScattering, &scatteringPdf, flagsNS, &sampledType);
        f = f * absdot(wi, bsdf.ns);
    }
    if (!is_black(f) && scatteringPdf > 0) {
        // light.Pdf_Li -> Shape::Pdf (shape.cpp:72-87): intersect the light's own triangle
        const V3 ro = offset_ray_origin(is.p, is.pError, is.n, wi);
        float lpdf = 0.f, tLight = 0.f;  // tLight: distance along the MIS ray to the light's own shape
        V3 ln = mk(0.f, 0.f, 0.f);
        TriHit h;
        if (onSphere) {
            // Sphere::Pdf (sphere.cpp:292-304); the ray can only return this light's radiance if it meets the sphere
            float th;
            Isect li;
            if (sphere_intersect(*lsp, ro, wi, pt_inf(), &th, &li)) {
                ln = li.n;
                tLight = th;
                lpdf = sphere_pdf(*lsp, is.p, is.pError, is.n, wi);
            } else if (general) {
                // from outside, Sphere::Pdf is the cone's density whether or not wi points into the cone: the reference
                // traces the ray (it finds no light); with bounded media its segments are counted, so it is traced here too
                lpdf = sphere_pdf(*lsp, is.p, is.pError, is.n, wi);
            }
        } else if (!ldegenerate && triangle_test(p0, p1, p2, ro, make_shear(wi), pt_inf(), &h)) {
            Isect li;
            fill_isect(p0, p1, p2, lflip, lsh, h, wi, &li);
            ln = li.n;
            tLight = h.t;
            lpdf = len2(is.p - li.p) / (absdot(ln, -wi) * light.area);
            if (pt_isinf(lpdf)) lpdf = 0.f;
        }
        if (lpdf != 0) {
            const float weight = power_heuristic(scatteringPdf, lpdf);
            // lightIsect.Le(-wi) if the closest hit along the ray is this light (integrator.cpp:205-209)
            const Spec Le = (light.two_sided || dot(ln, -wi) > 0) ? lemit : rgb1(0.f);
            // ... attenuated by the medium up to that hit (Scene::IntersectTr: ray.tMax is the hit distance by then)
            const Spec Tr = medium ? medium_tr(sigmaT, wi, tLight) : rgb1(1.f);
            out->B = is_black(Le) ? rgb1(0.f) : f * Le * Tr * weight / scatteringPdf;
            if (general) {  // Le and Tr belong to the hit the walk ends on
                out->B = f;
                out->wB = weight;
                out->pdfB = scatteringPdf;
            }
            out->mi_o = ro;
            out->mi_d = wi;
            out->pend |= PEND_BSDF;
        }
    }
}

// bounded media: the start of the two rays' walks (transmittance 1, the medium around the vertex) and the light sample
__device__ __forceinline__ void store_direct_general(const RenderDev *R, uint32_t slot, const DirectOut &d, int med) {
#if B200PT_MEDIA_GENERAL
    const float mbits = __uint_as_float((uint32_t)med);
    if (d.pend & PEND_LIGHT) {
        R->A2[slot] = make_float4(d.A2.c[0], d.A2.c[1], d.A2.c[2], d.pdfA);
        R->sh_tr[slot] = make_float4(1.f, 1.f, 1.f, mbits);
        R->sh_p1[slot] = f4(d.p1, 0.f);
        R->sh_p1e[slot] = f4(d.p1e, 0.f);
        R->sh_p1n[slot] = f4(d.p1n, 0.f);
    }
    if (d.pend & PEND_BSDF) R->mi_tr[slot] = make_float4(1.f, 1.f, 1.f, mbits);
#endif
}

// ------------------------------------------------------------------ path-vertex steps
// One copy of each step shared by the kernels that process a path vertex per lane: k_shade of either spectrum build,
// k_medium and k_medium_general.

// The path ray of a slot and the fields of its meta word (PathRec::o / PathRec::d)
struct PathVertex {
    V3 ro, rd;
    float etaScale;
    uint32_t meta;
    int bounces;
    bool specularBounce;
};
__device__ __forceinline__ PathVertex load_vertex(const PathRec &P) {
    const float4 o4 = P.o, d4 = P.d;
    PathVertex v;
    v.ro = v3(o4);
    v.rd = v3(d4);
    v.etaScale = o4.w;
    v.meta = __float_as_uint(d4.w);
    v.bounces = (int)((v.meta >> 16) & 0xffu);
    v.specularBounce = ((v.meta >> 24) & PF_SPECULAR) != 0;
    return v;
}
// the sampler of a path, continued at the dimension its meta word holds
__device__ __forceinline__ SobolStream sobol_stream(uint64_t index, uint32_t meta) {
    SobolStream st;
    st.index = index;
    st.dim = (int)(meta & 0xffffu);
    st.px = st.py = 0;  // only dimensions 0/1 depend on the pixel
    return st;
}
__device__ __forceinline__ uint32_t pack_meta(int dim, int bounces, bool specular) {
    return ((uint32_t)dim & 0xffffu) | ((uint32_t)bounces << 16) | ((specular ? (uint32_t)PF_SPECULAR : 0u) << 24);
}
// the meta word of a path that stays on its bounce (bounces and flags kept) after it spent sampler dimensions
__device__ __forceinline__ uint32_t meta_with_dim(uint32_t meta, int dim) { return (meta & 0xffff0000u) | ((uint32_t)dim & 0xffffu); }

// Re-derives the accepted closest hit P.hit of the path ray as a surface interaction: Shape::Intersect's values (t, b0,
// b1, b2, or the sphere's root) do not depend on tMax.  Fills the hit's material word and light id too, and with tg the
// geometric dpdu / dpdv and uv a texture lookup needs.
template <bool VTX>
__device__ __forceinline__ bool accepted_hit(const RenderDev *R, const PathRec &P, const V3 &ro, const V3 &rd, Isect *is, uint32_t *mflags,
                                             int *lightId, TexGeom *tg = nullptr) {
    const uint32_t ti = P.hit;
    bool found;
    if (VTX && is_sphere_hit(ti)) {
        const DevSphere *sp = R->scene.spheres + (ti & SPHERE_HIT_MASK);
        float th;
        found = sphere_intersect(*sp, ro, rd, pt_inf(), &th, is, tg);
        *mflags = sp->mat_flags;
        *lightId = sp->light_id;
    } else {
        const F4 *tp = R->scene.tris + (size_t)ti * 3;
        const F4 t0 = ld_f4(tp), t1 = ld_f4(tp + 1), t2 = ld_f4(tp + 2);
        const V3 p0 = v3(t0), p1 = v3(t1), p2 = v3(t2);
        *mflags = __float_as_uint(t1.w);
        *lightId = (int)__float_as_uint(t2.w);
        TriHit h;
        if (VTX && (*mflags & B200PT_TRI_INSTANCED)) {
            // a triangle of an instanced object: intersect in the object's space, bring the hit back
            const DevInstance *in = R->scene.instances + P.hit_inst;
            V3 o2, d2;
            float tm2;
            instance_ray(*in, ro, rd, pt_inf(), &o2, &d2, &tm2);
            found = triangle_test(p0, p1, p2, o2, make_shear(d2), pt_inf(), &h);
            if (found) {
                TriShading tsh;
                load_shading<VTX>(R->scene, ti, *mflags, &tsh);
                fill_isect(p0, p1, p2, (*mflags & B200PT_TRI_FLIP) != 0, tsh, h, d2, is);
                if (tg) triangle_tex_geom(p0, p1, p2, tsh, h, tg);
                instance_isect_to_world(*in, is, tg);
            }
        } else {
            found = triangle_test(p0, p1, p2, ro, make_shear(rd), pt_inf(), &h);
            if (found) {
                TriShading tsh;
                load_shading<VTX>(R->scene, ti, *mflags, &tsh);
                fill_isect(p0, p1, p2, (*mflags & B200PT_TRI_FLIP) != 0, tsh, h, rd, is);
                if (tg) triangle_tex_geom(p0, p1, p2, tsh, h, tg);
            }
        }
    }
    return found;
}
// Distance of the closest hit `ti` = P.hit along (ro, rd) -- ray.tMax after Scene::Intersect, infinity for a miss -- and
// the hit's material word.  (k_medium_general never meets an instanced triangle: render_create refuses bounded media in
// scenes with object instances.)
__device__ __forceinline__ float hit_distance(const RenderDev *R, const PathRec &P, uint32_t ti, const V3 &ro, const V3 &rd,
                                              uint32_t *mflags) {
    float tHit = pt_inf();
    *mflags = 0;
    if (ti == B200PT_MISS) return tHit;
    if (is_sphere_hit(ti)) {
        const DevSphere *sp = R->scene.spheres + (ti & SPHERE_HIT_MASK);
        float th;
        if (sphere_intersect(*sp, ro, rd, pt_inf(), &th, nullptr)) tHit = th;
        *mflags = sp->mat_flags;
    } else {
        const F4 *tp = R->scene.tris + (size_t)ti * 3;
        const F4 t0 = ld_f4(tp), t1 = ld_f4(tp + 1), t2 = ld_f4(tp + 2);
        *mflags = __float_as_uint(t1.w);
        V3 o2 = ro, d2 = rd;
        if (*mflags & B200PT_TRI_INSTANCED) {  // a triangle of an instanced object: same ray parameter in the object's space
            float tm2;
            instance_ray(R->scene.instances[P.hit_inst], ro, rd, pt_inf(), &o2, &d2, &tm2);
        }
        TriHit h;
        if (triangle_test(v3(t0), v3(t1), v3(t2), o2, make_shear(d2), pt_inf(), &h)) tHit = h.t;
    }
    return tHit;
}
// lightDistribution->Lookup(p) (path.cpp:115: the uniform / power table, or the table of p's voxel) and
// SampleDiscrete(u) on it (UniformSampleOneLight, integrator.cpp:85-106)
__device__ __forceinline__ int pick_light(const RenderDev *R, const V3 &p, float u, float *pickPdf) {
    const float *cdf = R->light_cdf, *func = R->light_func;
    float funcInt = R->light_func_int;
    if (R->grid.enabled) {
        const int vox = spatial_voxel(R->grid, p);
        cdf = R->sp_cdf + (size_t)vox * (R->n_lights + 1);
        func = R->sp_func + (size_t)vox * R->n_lights;
        funcInt = R->sp_func_int[vox];
    }
    return sample_discrete(cdf, func, funcInt, R->n_lights, u, pickPdf);
}
// MediumInteraction(ray(t), -ray.d, ...): no normal, no error bounds
__device__ __forceinline__ Isect medium_interaction(const V3 &ro, const V3 &rd, float t) {
    Isect mi;
    mi.p = ro + rd * t;
    mi.wo = -rd;
    mi.n = mi.ns = mk(0.f, 0.f, 0.f);
    mi.pError = mk(0.f, 0.f, 0.f);
    return mi;
}
// HomogeneousMedium::Sample (homogeneous.cpp:49-76) on an eager spectrum: the channel and the free-flight distance against
// the distance tHit of the hit, beta *= Tr [* sigma_s] / pdf.  Returns t; *sampledMedium: the path scatters at ray(t).
__device__ __forceinline__ float sample_medium_rgb(const Spec &sigmaT, const Spec &sigmaS, const V3 &rd, float tHit, float uChannel,
                                                   float uDist, Spec *beta, bool *sampledMedium) {
    const int channel = pt_mini((int)(uChannel * B200PT_NSPEC), B200PT_NSPEC - 1);
    const float dist = -pt_logf(1 - uDist) / sigmaT.c[channel];
    const float rdLen = len(rd);
    const float t = pt_min(dist / rdLen, tHit);
    *sampledMedium = t < tHit;
    Spec Tr;
    PT_UNROLL SPEC_FOR Tr.c[i_] = pt_expf((-sigmaT.c[i_]) * pt_min(t, PT_MAX_FLOAT) * rdLen);
    const Spec density = *sampledMedium ? (sigmaT * Tr) : Tr;
    float pdf = 0.f;
    SPEC_FOR pdf += density.c[i_];
    pdf *= 1 / (float)B200PT_NSPEC;
    if (pdf == 0) pdf = 1;
    *beta = *beta * (*sampledMedium ? (Tr * sigmaS / pdf) : (Tr / pdf));
    return t;
}
// Russian roulette (path.cpp:176-184) of a path whose rrMax = max(beta * etaScale) is below the threshold, with the
// sample u the caller drew for it: false ends the path, otherwise beta /= 1 - q.
__device__ __forceinline__ bool russian_roulette(float rrMax, float u, Spec *beta) {
    const float q = pt_max(.05f, 1 - rrMax);
    if (u < q) return false;
    *beta = *beta / (1 - q);
    return true;
}
// ... with beta streamed through the slot's 60 bins
__device__ __forceinline__ bool russian_roulette(float rrMax, float u, float4 *sBeta) {
    const float q = pt_max(.05f, 1 - rrMax);
    if (u < q) return false;
    const float dq = 1 - q;
#pragma unroll 5
    for (int q4 = 0; q4 < B200PT_NSPEC / 4; ++q4) {
        const float4 v = sBeta[q4];
        sBeta[q4] = make_float4(v.x / dq, v.y / dq, v.z / dq, v.w / dq);
    }
    return true;
}

// What a vertex leaves behind: its pending shadow and MIS rays (counters in the bounce's block qc) and the path itself
// if it goes on.  Every lane of the warp must call it (converged).
__device__ __forceinline__ void append_vertex_out(const RenderDev *R, uint32_t *qc, uint32_t *qc_next, uint32_t *q_next, uint32_t pend,
                                                  bool cont, uint32_t slot) {
    const uint32_t ps = warp_append(&qc[Q_SHADOW], (pend & PEND_LIGHT) != 0);
    if (pend & PEND_LIGHT) R->q_shadow[ps] = slot;
    const uint32_t pm = warp_append(&qc[Q_MIS], (pend & PEND_BSDF) != 0);
    if (pend & PEND_BSDF) R->q_mis[pm] = slot;
    const uint32_t pn = warp_append(qc_next, cont);
    if (cont) q_next[pn] = slot;
}

#if B200PT_NSPEC == 3
// whether any parameter of material `mi` is an image texture (RenderDev::tex_bind != nullptr)
__device__ __forceinline__ bool material_textured(const RenderDev *R, uint32_t mi) {
    const DevTexBind *tb = R->tex_bind + (size_t)mi * B200PT_TEX_SLOTS;
    bool any = false;
    for (int k = 0; k < B200PT_TEX_SLOTS; ++k) any |= tb[k].mip >= 0;
    return any;
}
// The uv derivatives of a textured hit.  Only camera rays carry differentials (every SpawnRay drops them, path.cpp:161,
// volpath.cpp:115-121): at bounce 0 the camera ray is rebuilt from the sample's pFilm and lens sample (dimensions 3-4) and
// counts as the path ray only if it is that ray bit for bit -- a ray that crossed a medium boundary was spawned anew.
__device__ __forceinline__ void textured_hit(const RenderDev *R, const PathRec &P, uint32_t slot, const PathVertex &v, const Isect &is,
                                             TexGeom *tg) {
    bool has_diff = false;
    V3 rdiff[4];
    if (v.bounces == 0) {
        const float2 pf = R->pfilm[slot];
        const float pFilm[2] = {pf.x, pf.y};
        SobolStream cs = sobol_stream(P.sobol, 3u);
        float ul[2];
        get2d(R->sampler, cs, ul);
        V3 o, d;
        float tMax;
        generate_camera_ray(R->camera, pFilm, ul, &o, &d, &tMax);
        has_diff = o.x == v.ro.x && o.y == v.ro.y && o.z == v.ro.z && d.x == v.rd.x && d.y == v.rd.y && d.z == v.rd.z;
        if (has_diff) camera_ray_differentials(R->camera, R->dx_camera, R->dy_camera, R->diff_scale, pFilm, ul, o, d, rdiff);
    }
    compute_differentials(is, has_diff, rdiff, tg);
}
// resident CTAs per SM the shading kernels are compiled for (4 -> 128 registers; A/B builds: 5 -> 96, 6 -> 80)
#ifndef B200PT_SHADE_MINCTAS
#define B200PT_SHADE_MINCTAS 4
#endif
template <int MAT, bool VTX>
__global__ void __launch_bounds__(128, B200PT_SHADE_MINCTAS) k_shade(const RenderDev *R, int bounce, uint32_t *work) {
    uint32_t *qc = &R->qcount[bounce * Q_PER_BOUNCE];
    const uint32_t n = qc[Q_MAT0 + MAT];
    const uint32_t *queue = R->q_mat[MAT];
    uint32_t *qc_next = &R->qcount[(bounce + 1) * Q_PER_BOUNCE + Q_PATH];
    uint32_t *q_next = R->q_path[(bounce + 1) & 1];
    uint32_t i;
    while (warp_fetch(work, n, &i)) {
        const bool active = i < n;
        bool cont = false;
        uint32_t pend = 0, slot = 0;
        if (active) {
            slot = queue[i];
            PathRec &P = R->path[slot];
            PathVertex v = load_vertex(P);
            float betaW, LW;
            Spec beta = ld_spec(P.beta, R->s_beta, slot, &betaW);
            Spec L = ld_spec(P.L, R->s_L, slot, &LW);
            Isect is;
            uint32_t mflags;
            int lightId;
            TexGeom tg;
            const bool textures = VTX && R->tex_bind != nullptr;
            if (accepted_hit<VTX>(R, P, v.ro, v.rd, &is, &mflags, &lightId, textures ? &tg : nullptr)) {
                // path.cpp:91-101: emitted light at the first vertex or after a specular bounce
                if (v.bounces == 0 || v.specularBounce) {
                    if (lightId >= 0) {
                        const DevLight lt = R->lights[lightId];
                        const Spec Le = (lt.two_sided || dot(is.n, -v.rd) > 0) ? light_emit(R, lightId, lt) : rgb1(0.f);
                        L = L + beta * Le;
                    }
                }
                if (v.bounces < R->max_depth) {  // path.cpp:104
                    Bsdf bsdf;
                    const uint32_t mi = mflags & 0xffffu;
                    const b200pt_material *mat = &R->scene.materials[mi];
                    b200pt_material texMat;
                    if (textures && material_textured(R, mi)) {
                        texMat = *mat;
                        textured_hit(R, P, slot, v, is, &tg);
                        textured_material(R, mi, tg, &texMat);
                        mat = &texMat;
                    }
                    make_bsdf<MAT>(*mat, R->scene.material_spectra + (size_t)mi * (5 * B200PT_NSPEC), is, &bsdf);
                    SobolStream st = sobol_stream(P.sobol, v.meta);
                    const SamplerParams &sp = R->sampler;
                    // path.cpp:119-128 -> UniformSampleOneLight (integrator.cpp:85-106)
                    // (VolPathIntegrator samples a light at every surface vertex, volpath.cpp:124-128)
                    if (((VTX && R->volpath) || bsdf_num_components(bsdf, BSDF_ALL & ~BSDF_SPECULAR) > 0) && R->n_lights > 0) {
                        float pickPdf;
                        const int lightNum = pick_light(R, is.p, get1d(sp, st), &pickPdf);
                        if (pickPdf != 0) {
                            float uLight[2], uScattering[2];
                            get2d(sp, st, uLight);
                            get2d(sp, st, uScattering);
                            DirectOut dout;
                            const int med = (B200PT_MEDIA_GENERAL && VTX && R->med_general) ? R->cur_med[slot] : 0;
                            estimate_direct<VTX, mat_kinds(MAT)>(R, is, bsdf, uScattering, lightNum, uLight, &dout, false, med);
                            pend = dout.pend;
                            // without pending rays nothing is stored: k_resolve left the pending flags at 0
                            if (pend) {
                                DirectRec &D = R->direct[slot];
                                D.sh_o = f4(dout.sh_o, __uint_as_float((uint32_t)lightNum));
                                D.sh_d = f4(dout.sh_d, __uint_as_float(pend));
                                if (pend & PEND_BSDF) {
                                    D.mi_o = f4(dout.mi_o, dout.pdfB);
                                    D.mi_d = f4(dout.mi_d, 0.f);
                                }
                                // A and B share a sector: both are stored (the one not pending is never read)
                                st_spec(D.A, R->s_A, slot, dout.A, dout.wA);
                                st_spec(D.B, R->s_B, slot, dout.B, dout.wB);
                                st_beta_ld(D, R->s_beta_ld, slot, beta, pickPdf);
                                if (B200PT_MEDIA_GENERAL && VTX && R->med_general) store_direct_general(R, slot, dout, med);
                            }
                        }
                    }
                    // path.cpp:131-150: sample the BSDF for the next direction
                    const V3 wo = -v.rd;
                    V3 wi = mk(0.f, 0.f, 0.f);
                    float pdf = 0.f;
                    int flags = 0;
                    float u2[2];
                    get2d(sp, st, u2);
                    const Spec f = bsdf_sample_f<mat_kinds(MAT)>(bsdf, wo, &wi, u2, &pdf, BSDF_ALL, &flags);
                    if (!(is_black(f) || pdf == 0.f)) {
                        beta = beta * (f * absdot(wi, bsdf.ns) / pdf);
                        const bool spec = (flags & BSDF_SPECULAR) != 0;
                        if ((flags & BSDF_SPECULAR) && (flags & BSDF_TRANSMISSION)) {
                            const float eta = bsdf.eta;
                            v.etaScale *= (dot(wo, is.n) > 0) ? (eta * eta) : 1 / (eta * eta);
                        }
                        const V3 no = offset_ray_origin(is.p, is.pError, is.n, wi);  // isect.SpawnRay(wi)
                        cont = true;
                        const float rrMax = max_comp(beta * v.etaScale);
                        if (rrMax < R->rr_threshold && v.bounces > 3) cont = russian_roulette(rrMax, get1d(sp, st), &beta);
                        if (cont) {
                            P.o = f4(no, v.etaScale);
                            P.d = f4(wi, __uint_as_float(pack_meta(st.dim, v.bounces + 1, spec)));
                            betaW = 0.f;
                        }
                    }
                }
                // beta and L share a sector: both are stored (the beta of a path that ends here is never read)
                st_spec(P.beta, R->s_beta, slot, beta, betaW);
                st_spec(P.L, R->s_L, slot, L, LW);
            }
        }
        append_vertex_out(R, qc, qc_next, q_next, pend, cont, slot);
    }
}

#else
// ---- SampledSpectrum build: the same vertex with lazy spectra (pt_core.cuh "Lazy spectra").  No Spec by value: the
// BSDF value is a recipe (FSpec), the light's radiance a row of the light table with a few scalars (LiTerm), and beta,
// beta_ld, A, B and L are streamed bin by bin between the slot-major per-slot arrays -- the arithmetic per bin is that of the
// eager kernel above / estimate_direct, operation for operation.
struct LiTerm {
    const float *row;  // nullptr: black
    int op;            // 1: row   2: row / s0   3: (row * s0) / s1
    float s0, s1;
    const float *sigma_t;  // != nullptr: times Exp(-sigma_t * x) (homogeneous medium around the scene)
    float x;
};
__device__ __forceinline__ void li_eval4(const LiTerm &t, int b0, float v[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float r = t.row[b0 + j];
        float li = t.op == 1 ? r : (t.op == 2 ? r / t.s0 : (r * t.s0) / t.s1);
        if (t.sigma_t) li = li * pt_expf((-t.sigma_t[b0 + j]) * t.x);
        v[j] = li;
    }
}
__device__ __forceinline__ bool li_is_black(const LiTerm &t) {
    if (!t.row) return true;
    for (int b0 = 0; b0 < B200PT_NSPEC; b0 += 4) {
        float v[4];
        LiTerm u = t;
        u.sigma_t = nullptr;  // callers test Li before the transmittance is applied
        li_eval4(u, b0, v);
        if (v[0] != 0.f || v[1] != 0.f || v[2] != 0.f || v[3] != 0.f) return false;
    }
    return true;
}
struct DirectLazy {
    uint32_t pend;
    V3 sh_o, sh_d, mi_o, mi_d;
};
// estimate_direct with the two terms written straight into the slot's A / B rows
template <int KINDS, bool inMedium = false>
__device__ void estimate_direct_lazy(const RenderDev *R, uint32_t slot, const Isect &is, const Bsdf &bsdf, const float uScattering[2],
                                     int lightNum, const float uLight[2], DirectLazy *out) {
    // inMedium: `is` is a MediumInteraction and the Henyey-Greenstein phase function takes the BSDF's place (its value p is
    // the constant spectrum Spectrum(p) and there is no cosine: |cos| = 1 multiplies exactly)
    const float hgG = R->med_g;
    const bool medium = R->has_medium != 0;
    const float *sigmaT = medium ? R->med_spectra + B200PT_NSPEC : nullptr;
    float4 *sA = reinterpret_cast<float4 *>(R->s_A + (size_t)slot * B200PT_NSPEC);
    float4 *sB = reinterpret_cast<float4 *>(R->s_B + (size_t)slot * B200PT_NSPEC);
    out->pend = 0;
    out->sh_o = out->sh_d = out->mi_o = out->mi_d = mk(0.f, 0.f, 0.f);
    const DevLight &lightRef = R->lights[lightNum];
    const float *lrow = R->light_spectra + (size_t)lightNum * B200PT_NSPEC;
    if (lightRef.kind != 0) {
        // delta light: delta_light_sample (pt_sphere.cuh) as a recipe
        const V3 lpos = mk(lightRef.position[0], lightRef.position[1], lightRef.position[2]);
        V3 wiD, pTarget;
        LiTerm Li;
        Li.row = lrow;
        Li.sigma_t = nullptr;
        Li.x = 0.f;
        Li.s0 = Li.s1 = 0.f;
        if (lightRef.kind == 3) {
            wiD = lpos;
            pTarget = is.p + lpos * lightRef.two_world_radius;
            Li.op = 1;
        } else {
            wiD = normalize(lpos - is.p);
            pTarget = lpos;
            const float d2 = len2(lpos - is.p);
            if (lightRef.kind == 1) {
                Li.op = 2;
                Li.s0 = d2;
            } else {
                const V3 wl = normalize(xform_vector(lightRef.world_to_light, -wiD));
                const float cosTheta = wl.z;
                float falloff;
                if (cosTheta < lightRef.cos_total_width)
                    falloff = 0.f;
                else if (cosTheta >= lightRef.cos_falloff_start)
                    falloff = 1.f;
                else {
                    const float delta = (cosTheta - lightRef.cos_total_width) / (lightRef.cos_falloff_start - lightRef.cos_total_width);
                    falloff = (delta * delta) * (delta * delta);
                }
                Li.op = 3;
                Li.s0 = falloff;
                Li.s1 = d2;
            }
        }
        if (!li_is_black(Li)) {
            const FSpec fD = inMedium ? fspec_const(phase_hg(dot(is.wo, wiD), hgG))
                                      : bsdf_f_lazy<KINDS>(bsdf, is.wo, wiD, BSDF_ALL & ~BSDF_SPECULAR);
            const float ad = inMedium ? 1.f : absdot(wiD, bsdf.ns);
            if (!fspec_is_black<KINDS>(fD, ad)) {
                const V3 origin = offset_ray_origin(is.p, is.pError, is.n, pTarget - is.p);
                out->sh_o = origin;
                out->sh_d = pTarget - origin;
                if (medium) {
                    Li.sigma_t = sigmaT;
                    Li.x = pt_min(PT_SHADOW_TMAX * len(out->sh_d), PT_MAX_FLOAT);
                }
#pragma unroll 1
                for (int b0 = 0; b0 < B200PT_NSPEC; b0 += 4) {
                    float fv[4], lv[4];
                    fspec_eval4<KINDS>(fD, b0, fv);
                    li_eval4(Li, b0, lv);
                    sA[b0 >> 2] = make_float4(((fv[0] * ad) * lv[0]) / 1.f, ((fv[1] * ad) * lv[1]) / 1.f, ((fv[2] * ad) * lv[2]) / 1.f,
                                              ((fv[3] * ad) * lv[3]) / 1.f);
                }
                out->pend |= PEND_LIGHT;
            }
        }
        return;
    }
    const DevLight light = lightRef;
    const bool onSphere = is_sphere_hit(light.tri);
    const DevSphere *lsp = onSphere ? R->scene.spheres + (light.tri & SPHERE_HIT_MASK) : nullptr;
    const F4 *tp = R->scene.tris + (size_t)(onSphere ? 0u : light.tri) * 3;
    F4 t0 = {0.f, 0.f, 0.f, 0.f}, t1 = t0, t2 = t0;
    if (!onSphere) {
        t0 = ld_f4(tp);
        t1 = ld_f4(tp + 1);
        t2 = ld_f4(tp + 2);
    }
    const V3 p0 = v3(t0), p1 = v3(t1), p2 = v3(t2);
    const uint32_t lflags = __float_as_uint(t1.w);
    const bool lflip = (lflags & B200PT_TRI_FLIP) != 0, ldegenerate = (lflags & B200PT_TRI_DEGENERATE) != 0;
    TriShading lsh;
    load_shading<true>(R->scene, light.tri, lflags, &lsh);
    const int flagsNS = BSDF_ALL & ~BSDF_SPECULAR;
    V3 wi = mk(0.f, 0.f, 0.f);
    float lightPdf = 0.f, scatteringPdf = 0.f;
    LiTerm Li;
    Li.row = nullptr;
    Li.op = 1;
    Li.s0 = Li.s1 = Li.x = 0.f;
    Li.sigma_t = nullptr;
    LightSample ps;
    if (onSphere) {
        ps = sphere_sample(*lsp, is.p, is.pError, is.n, uLight, &lightPdf);
    } else {
        ps = triangle_sample(p0, p1, p2, lflip, lsh, uLight, &lightPdf);
        V3 w = ps.p - is.p;
        if (len2(w) == 0)
            lightPdf = 0;
        else {
            w = normalize(w);
            lightPdf *= len2(is.p - ps.p) / absdot(ps.n, -w);
            if (pt_isinf(lightPdf)) lightPdf = 0.f;
        }
    }
    if (lightPdf == 0 || len2(ps.p - is.p) == 0) {
        lightPdf = 0;
    } else {
        wi = normalize(ps.p - is.p);
        Li.row = (light.two_sided || dot(ps.n, -wi) > 0) ? lrow : nullptr;
    }
    if (lightPdf > 0 && !li_is_black(Li)) {
        FSpec f;
        float ad = 1.f;
        if (inMedium) {
            const float p = phase_hg(dot(is.wo, wi), hgG);
            f = fspec_const(p);
            scatteringPdf = p;
        } else {
            f = bsdf_f_lazy<KINDS>(bsdf, is.wo, wi, flagsNS);
            ad = absdot(wi, bsdf.ns);
            scatteringPdf = bsdf_pdf<KINDS>(bsdf, is.wo, wi, flagsNS);
        }
        if (!fspec_is_black<KINDS>(f, ad)) {
            const V3 origin = offset_ray_origin(is.p, is.pError, is.n, ps.p - is.p);
            const V3 target = offset_ray_origin(ps.p, ps.pError, ps.n, origin - ps.p);
            out->sh_o = origin;
            out->sh_d = target - origin;
            if (medium) {
                Li.sigma_t = sigmaT;
                Li.x = pt_min(PT_SHADOW_TMAX * len(out->sh_d), PT_MAX_FLOAT);
            }
            const float weight = power_heuristic(lightPdf, scatteringPdf);
#pragma unroll 1
            for (int b0 = 0; b0 < B200PT_NSPEC; b0 += 4) {
                float fv[4], lv[4];
                fspec_eval4<KINDS>(f, b0, fv);
                li_eval4(Li, b0, lv);
                float av[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) av[j] = (((fv[j] * ad) * lv[j]) * weight) / lightPdf;
                sA[b0 >> 2] = make_float4(av[0], av[1], av[2], av[3]);
            }
            out->pend |= PEND_LIGHT;
        }
    }
    // BSDF sampling with MIS
    int sampledType = 0;
    FSpec f;
    float ad = 1.f;
    if (inMedium) {
        const float p = hg_sample_p(hgG, is.wo, &wi, uScattering);
        f = fspec_const(p);
        scatteringPdf = p;
    } else {
        f = bsdf_sample_f_lazy<KINDS>(bsdf, is.wo, &wi, uScattering, &scatteringPdf, flagsNS, &sampledType);
        ad = absdot(wi, bsdf.ns);
    }
    if (!fspec_is_black<KINDS>(f, ad) && scatteringPdf > 0) {
        const V3 ro = offset_ray_origin(is.p, is.pError, is.n, wi);
        float lpdf = 0.f, tLight = 0.f;
        V3 ln = mk(0.f, 0.f, 0.f);
        TriHit h;
        if (onSphere) {
            float th;
            Isect li;
            if (sphere_intersect(*lsp, ro, wi, pt_inf(), &th, &li)) {
                ln = li.n;
                tLight = th;
                lpdf = sphere_pdf(*lsp, is.p, is.pError, is.n, wi);
            }
        } else if (!ldegenerate && triangle_test(p0, p1, p2, ro, make_shear(wi), pt_inf(), &h)) {
            Isect li;
            fill_isect(p0, p1, p2, lflip, lsh, h, wi, &li);
            ln = li.n;
            tLight = h.t;
            lpdf = len2(is.p - li.p) / (absdot(ln, -wi) * light.area);
            if (pt_isinf(lpdf)) lpdf = 0.f;
        }
        if (lpdf != 0) {
            const float weight = power_heuristic(scatteringPdf, lpdf);
            LiTerm Le;
            Le.row = (light.two_sided || dot(ln, -wi) > 0) ? lrow : nullptr;
            Le.op = 1;
            Le.s0 = Le.s1 = 0.f;
            Le.sigma_t = nullptr;
            Le.x = 0.f;
            const bool black = li_is_black(Le);
            const float xTr = medium ? pt_min(tLight * len(wi), PT_MAX_FLOAT) : 0.f;
#pragma unroll 1
            for (int b0 = 0; b0 < B200PT_NSPEC; b0 += 4) {
                float fv[4], lv[4];
                if (!black) {
                    fspec_eval4<KINDS>(f, b0, fv);
                    li_eval4(Le, b0, lv);
                }
                float bv[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float bval = 0.f;
                    if (!black) {
                        const float tr = medium ? pt_expf((-sigmaT[b0 + j]) * xTr) : 1.f;
                        bval = ((((fv[j] * ad) * lv[j]) * tr) * weight) / scatteringPdf;
                    }
                    bv[j] = bval;
                }
                sB[b0 >> 2] = make_float4(bv[0], bv[1], bv[2], bv[3]);
            }
            out->mi_o = ro;
            out->mi_d = wi;
            out->pend |= PEND_BSDF;
        }
    }
}

// resident CTAs per SM the 60-bin shading kernel is compiled for (register budget: 4 -> 128, 3 -> 168, 2 -> 255)
#ifndef B200PT_S60_SHADE_MINCTAS
#define B200PT_S60_SHADE_MINCTAS 4
#endif
template <int MAT, bool VTX>
__global__ void __launch_bounds__(128, B200PT_S60_SHADE_MINCTAS) k_shade(const RenderDev *R, int bounce, uint32_t *work) {
    uint32_t *qc = &R->qcount[bounce * Q_PER_BOUNCE];
    const uint32_t n = qc[Q_MAT0 + MAT];
    const uint32_t *queue = R->q_mat[MAT];
    uint32_t *qc_next = &R->qcount[(bounce + 1) * Q_PER_BOUNCE + Q_PATH];
    uint32_t *q_next = R->q_path[(bounce + 1) & 1];
    uint32_t i;
    while (warp_fetch(work, n, &i)) {
        const bool active = i < n;
        bool cont = false;
        uint32_t pend = 0, slot = 0;
        if (active) {
            slot = queue[i];
            PathRec &P = R->path[slot];
            PathVertex v = load_vertex(P);
            float4 *sBeta = reinterpret_cast<float4 *>(R->s_beta + (size_t)slot * B200PT_NSPEC);
            float4 *sL = reinterpret_cast<float4 *>(R->s_L + (size_t)slot * B200PT_NSPEC);
            Isect is;
            uint32_t mflags;
            int lightId;
            if (accepted_hit<true>(R, P, v.ro, v.rd, &is, &mflags, &lightId)) {
                // path.cpp:91-101: L += beta * Le at the first vertex or after a specular bounce
                if ((v.bounces == 0 || v.specularBounce) && lightId >= 0) {
                    const DevLight &lt = R->lights[lightId];
                    if (lt.two_sided || dot(is.n, -v.rd) > 0) {
                        const float *le = R->light_spectra + (size_t)lightId * B200PT_NSPEC;
#pragma unroll 3
                        for (int q = 0; q < B200PT_NSPEC / 4; ++q) {
                            const float4 l = sL[q], bt = sBeta[q];
                            sL[q] = make_float4(l.x + bt.x * le[4 * q], l.y + bt.y * le[4 * q + 1], l.z + bt.z * le[4 * q + 2],
                                                l.w + bt.w * le[4 * q + 3]);
                        }
                    } else {
                        // L + beta * 0: only a -0 would change, and L never holds one (it starts at +0 and only sums)
                    }
                }
                if (v.bounces < R->max_depth) {
                    Bsdf bsdf;
                    const uint32_t mi = mflags & 0xffffu;
                    make_bsdf<MAT>(R->scene.materials[mi], R->scene.material_spectra + (size_t)mi * (5 * B200PT_NSPEC), is, &bsdf);
                    SobolStream st = sobol_stream(P.sobol, v.meta);
                    const SamplerParams &sp = R->sampler;
                    if ((R->volpath || bsdf_num_components(bsdf, BSDF_ALL & ~BSDF_SPECULAR) > 0) && R->n_lights > 0) {
                        float pickPdf;
                        const int lightNum = pick_light(R, is.p, get1d(sp, st), &pickPdf);
                        if (pickPdf != 0) {
                            float uLight[2], uScattering[2];
                            get2d(sp, st, uLight);
                            get2d(sp, st, uScattering);
                            DirectLazy dout;
                            estimate_direct_lazy<mat_kinds(MAT)>(R, slot, is, bsdf, uScattering, lightNum, uLight, &dout);
                            pend = dout.pend;
                            // without pending rays nothing is stored: k_resolve left the pending flags at 0
                            if (pend) {
                                // beta as it is before this vertex's BSDF sample scales it
                                float4 *sBl = reinterpret_cast<float4 *>(R->s_beta_ld + (size_t)slot * B200PT_NSPEC);
#pragma unroll 5
                                for (int q = 0; q < B200PT_NSPEC / 4; ++q) sBl[q] = sBeta[q];
                                DirectRec &D = R->direct[slot];
                                D.sh_o = f4(dout.sh_o, __uint_as_float((uint32_t)lightNum));
                                D.sh_d = f4(dout.sh_d, __uint_as_float(pend));
                                if (pend & PEND_BSDF) {
                                    D.mi_o = f4(dout.mi_o, 0.f);
                                    D.mi_d = f4(dout.mi_d, 0.f);
                                }
                                D.A = make_float4(0.f, 0.f, 0.f, 0.f);
                                D.B = make_float4(0.f, 0.f, 0.f, 0.f);
                                D.beta_ld = make_float4(0.f, 0.f, 0.f, pickPdf);
                                reset_direct_hits(D);
                            }
                        }
                    }
                    // path.cpp:131-150
                    const V3 wo = -v.rd;
                    V3 wi = mk(0.f, 0.f, 0.f);
                    float pdf = 0.f;
                    int flags = 0;
                    float u2[2];
                    get2d(sp, st, u2);
                    const FSpec f = bsdf_sample_f_lazy<mat_kinds(MAT)>(bsdf, wo, &wi, u2, &pdf, BSDF_ALL, &flags);
                    if (!(fspec_is_black<mat_kinds(MAT)>(f, 1.f) || pdf == 0.f)) {
                        const float ad = absdot(wi, bsdf.ns);
                        const bool spec = (flags & BSDF_SPECULAR) != 0;
                        if ((flags & BSDF_SPECULAR) && (flags & BSDF_TRANSMISSION)) {
                            const float eta = bsdf.eta;
                            v.etaScale *= (dot(wo, is.n) > 0) ? (eta * eta) : 1 / (eta * eta);
                        }
                        const V3 no = offset_ray_origin(is.p, is.pError, is.n, wi);
                        cont = true;
                        // beta *= f * |cos| / pdf, and max(beta * etaScale) for the roulette (path.cpp:176-184)
                        float mx = 0.f;
#pragma unroll 1
                        for (int b0 = 0; b0 < B200PT_NSPEC; b0 += 4) {
                            float fv[4];
                            fspec_eval4<mat_kinds(MAT)>(f, b0, fv);
                            const float4 bo = sBeta[b0 >> 2];
                            const float bold[4] = {bo.x, bo.y, bo.z, bo.w};
                            float nbv[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const float nb = bold[j] * ((fv[j] * ad) / pdf);
                                nbv[j] = nb;
                                const float rr = nb * v.etaScale;
                                mx = (b0 + j == 0) ? rr : pt_max(mx, rr);
                            }
                            sBeta[b0 >> 2] = make_float4(nbv[0], nbv[1], nbv[2], nbv[3]);
                        }
                        if (mx < R->rr_threshold && v.bounces > 3) cont = russian_roulette(mx, get1d(sp, st), sBeta);
                        if (cont) {
                            P.o = f4(no, v.etaScale);
                            P.d = f4(wi, __uint_as_float(pack_meta(st.dim, v.bounces + 1, spec)));
                            P.beta = make_float4(0.f, 0.f, 0.f, 0.f);
                        }
                    }
                }
            }
        }
        append_vertex_out(R, qc, qc_next, q_next, pend, cont, slot);
    }
}
#endif  // B200PT_NSPEC == 3 (k_shade)

// Medium pass of a bounce (VolPathIntegrator with every ray inside one homogeneous medium, volpath.cpp:77-103): runs over
// the bounce's path rays after the closest-hit launch (which then does not classify).  It draws the channel and the
// free-flight distance (HomogeneousMedium::Sample, homogeneous.cpp:49-76) against the distance of the hit.  A path that
// scatters in the medium gets its whole vertex here -- light sample with the phase function, phase-sampled MIS ray and
// next direction, Russian roulette -- and skips the shading kernels; the others have beta scaled by Tr / pdf and are
// appended to their BSDF family's queue (rays that left the scene end here, like in the reference).
__global__ void __launch_bounds__(128, 4) k_medium(const RenderDev *R, int bounce, uint32_t *work) {
    const uint32_t n = R->qcount[bounce * Q_PER_BOUNCE + Q_PATH];
    const uint32_t *queue = R->q_path[bounce & 1];
    uint32_t *qc = &R->qcount[bounce * Q_PER_BOUNCE];
    uint32_t *qc_next = &R->qcount[(bounce + 1) * Q_PER_BOUNCE + Q_PATH];
    uint32_t *q_next = R->q_path[(bounce + 1) & 1];
#if B200PT_NSPEC == 3
    const Spec sigmaT = medium_sigma_t(R), sigmaS = medium_sigma_s(R);
#else
    // 60 bins: the medium's rows are read in place and beta is streamed through the slot's row (lazy spectra, see k_shade)
    const float *sigmaSrow = R->med_spectra, *sigmaTrow = R->med_spectra + B200PT_NSPEC;
#endif
    uint32_t i;
    while (warp_fetch(work, n, &i)) {
        const bool active = i < n;
        bool cont = false;
        int family = -1;
        uint32_t pend = 0, slot = 0;
        if (active) {
            slot = queue[i];
            PathRec &P = R->path[slot];
            const PathVertex v = load_vertex(P);
#if B200PT_NSPEC == 3
            float betaW;
            Spec beta = ld_spec(P.beta, R->s_beta, slot, &betaW);
#else
            const float betaW = P.beta.w;
            float4 *sBeta = reinterpret_cast<float4 *>(R->s_beta + (size_t)slot * B200PT_NSPEC);
#endif
            const uint32_t ti = P.hit;
            uint32_t mflags;
            const float tHit = hit_distance(R, P, ti, v.ro, v.rd, &mflags);
            SobolStream st = sobol_stream(P.sobol, v.meta);
            const SamplerParams &sp = R->sampler;
            // HomogeneousMedium::Sample
            const float uChannel = get1d(sp, st), uDist = get1d(sp, st);
#if B200PT_NSPEC == 3
            bool sampledMedium;
            const float t = sample_medium_rgb(sigmaT, sigmaS, v.rd, tHit, uChannel, uDist, &beta, &sampledMedium);
            const bool alive = !is_black(beta);
#else
            const int channel = pt_mini((int)(uChannel * B200PT_NSPEC), B200PT_NSPEC - 1);
            const float dist = -pt_logf(1 - uDist) / sigmaTrow[channel];
            const float rdLen = len(v.rd);
            const float t = pt_min(dist / rdLen, tHit);
            const bool sampledMedium = t < tHit;
            // two passes over the bins: the pdf (mean density), then beta *= Tr [* sigma_s] / pdf with the is_black test
            const float tClamped = pt_min(t, PT_MAX_FLOAT);
            float pdf = 0.f;
#pragma unroll 4
            for (int b = 0; b < B200PT_NSPEC; ++b) {
                const float tr = pt_expf((-sigmaTrow[b]) * tClamped * rdLen);
                pdf += sampledMedium ? (sigmaTrow[b] * tr) : tr;
            }
            pdf *= 1 / (float)B200PT_NSPEC;
            if (pdf == 0) pdf = 1;
            bool alive = false;
#pragma unroll 1
            for (int q = 0; q < B200PT_NSPEC / 4; ++q) {
                const float4 bo = sBeta[q];
                const float bold[4] = {bo.x, bo.y, bo.z, bo.w};
                float nb[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int b = 4 * q + j;
                    const float tr = pt_expf((-sigmaTrow[b]) * tClamped * rdLen);
                    nb[j] = bold[j] * (sampledMedium ? ((tr * sigmaSrow[b]) / pdf) : (tr / pdf));
                    alive = alive || nb[j] != 0.f;
                }
                sBeta[q] = make_float4(nb[0], nb[1], nb[2], nb[3]);
            }
#endif
            if (alive) {
                if (!sampledMedium) {
                    // on to the surface vertex (or out of the scene)
#if B200PT_NSPEC == 3
                    st_spec(P.beta, R->s_beta, slot, beta, betaW);
#else
                    P.beta = make_float4(0.f, 0.f, 0.f, betaW);
#endif
                    P.d = f4(v.rd, __uint_as_float(meta_with_dim(v.meta, st.dim)));
                    if (ti != B200PT_MISS) family = hit_family(R->scene.materials, mflags);
                } else if (v.bounces < R->max_depth) {  // volpath.cpp:84-85
                    const Isect mi = medium_interaction(v.ro, v.rd, t);
                    if (R->n_lights > 0) {
                        // UniformSampleOneLight(mi, ..., handleMedia = true), integrator.cpp:85-106
                        float pickPdf;
                        const int lightNum = pick_light(R, mi.p, get1d(sp, st), &pickPdf);
                        if (pickPdf != 0) {
                            float uLight[2], uScattering[2];
                            get2d(sp, st, uLight);
                            get2d(sp, st, uScattering);
                            Bsdf none;
                            none.n = 0;
#if B200PT_NSPEC == 3
                            DirectOut dout;
                            estimate_direct<true>(R, mi, none, uScattering, lightNum, uLight, &dout, true);
                            pend = dout.pend;
                            if (pend) {
                                st_beta_ld(R->direct[slot], R->s_beta_ld, slot, beta, pickPdf);
                                R->direct[slot].sh_o = f4(dout.sh_o, __uint_as_float((uint32_t)lightNum));
                                if (pend & PEND_LIGHT) st_spec(R->direct[slot].A, R->s_A, slot, dout.A, 0.f);
                                if (pend & PEND_BSDF) {
                                    R->direct[slot].mi_o = f4(dout.mi_o, 0.f);
                                    R->direct[slot].mi_d = f4(dout.mi_d, 0.f);
                                    st_spec(R->direct[slot].B, R->s_B, slot, dout.B, 0.f);
                                }
                            }
#else
                            DirectLazy dout;
                            estimate_direct_lazy<KM_CONST, true>(R, slot, mi, none, uScattering, lightNum, uLight, &dout);
                            pend = dout.pend;
                            if (pend) {
                                float4 *sBl = reinterpret_cast<float4 *>(R->s_beta_ld + (size_t)slot * B200PT_NSPEC);
#pragma unroll 5
                                for (int q = 0; q < B200PT_NSPEC / 4; ++q) sBl[q] = sBeta[q];
                                R->direct[slot].beta_ld = make_float4(0.f, 0.f, 0.f, pickPdf);
                                reset_direct_hits(R->direct[slot]);
                                R->direct[slot].sh_o = f4(dout.sh_o, __uint_as_float((uint32_t)lightNum));
                                if (pend & PEND_LIGHT) R->direct[slot].A = make_float4(0.f, 0.f, 0.f, 0.f);
                                if (pend & PEND_BSDF) {
                                    R->direct[slot].mi_o = f4(dout.mi_o, 0.f);
                                    R->direct[slot].mi_d = f4(dout.mi_d, 0.f);
                                    R->direct[slot].B = make_float4(0.f, 0.f, 0.f, 0.f);
                                }
                            }
#endif
                            R->direct[slot].sh_d = f4(dout.sh_d, __uint_as_float(pend));
                        }
                    }
                    // mi.phase->Sample_p(wo, &wi, sampler.Get2D()); ray = mi.SpawnRay(wi) (volpath.cpp:95-98)
                    V3 wi;
                    float u2[2];
                    get2d(sp, st, u2);
                    hg_sample_p(R->med_g, mi.wo, &wi, u2);
                    const V3 no = offset_ray_origin(mi.p, mi.pError, mi.n, wi);
                    cont = true;
#if B200PT_NSPEC == 3
                    const float rrMax = max_comp(beta * v.etaScale);  // volpath.cpp:176-184
                    if (rrMax < R->rr_threshold && v.bounces > 3) cont = russian_roulette(rrMax, get1d(sp, st), &beta);
#else
                    if (v.bounces > 3) {  // volpath.cpp:176-184 (the maximum is only needed then)
                        float mx = 0.f;
#pragma unroll 3
                        for (int q4 = 0; q4 < B200PT_NSPEC / 4; ++q4) {
                            const float4 b = sBeta[q4];
                            const float r0 = b.x * v.etaScale, r1 = b.y * v.etaScale, r2 = b.z * v.etaScale, r3 = b.w * v.etaScale;
                            mx = q4 == 0 ? r0 : pt_max(mx, r0);
                            mx = pt_max(pt_max(pt_max(mx, r1), r2), r3);
                        }
                        if (mx < R->rr_threshold) cont = russian_roulette(mx, get1d(sp, st), sBeta);
                    }
#endif
                    if (cont) {
                        P.o = f4(no, v.etaScale);
                        P.d = f4(wi, __uint_as_float(pack_meta(st.dim, v.bounces + 1, false)));
#if B200PT_NSPEC == 3
                        st_spec(P.beta, R->s_beta, slot, beta, 0.f);
#else
                        P.beta = make_float4(0.f, 0.f, 0.f, 0.f);
#endif
                    }
                }
            }
        }
        append_family(R->q_mat, &qc[Q_MAT0], family, slot);
        append_vertex_out(R, qc, qc_next, q_next, pend, cont, slot);
    }
}

#if B200PT_MEDIA_GENERAL
// ---- media bounded by null-material spheres (b200pt_integrator_desc::bounded_media) ------------------------------------
// medium id inside the boundary sphere that hit `ti` names, -1 when the hit is an ordinary surface (or a miss)
__device__ __forceinline__ int boundary_medium(const RenderDev *R, uint32_t ti) {
    return (ti != B200PT_MISS && is_sphere_hit(ti)) ? R->sphere_med[ti & SPHERE_HIT_MASK] : -1;
}

// The medium pass of k_medium for scenes whose media are bounded by surfaces (volpath.cpp:77-121).  Differences: the ray's
// medium is per-path state (cur_med; vacuum samples nothing and spends no sampler dimension), and a ray that reaches a
// boundary -- a surface without a BSDF -- continues behind it in the medium of the side it leaves on (interaction.h:80-82)
// without spending a bounce: it goes to q_cross and is traced again before the bounce's shading kernels run.
__global__ void __launch_bounds__(128, 4) k_medium_general(const RenderDev *R, int bounce, const uint32_t *queue, const uint32_t *count,
                                                           uint32_t *q_cross, uint32_t *cross_count, uint32_t *work, int count_rays) {
    const uint32_t n = *count;
    if (count_rays && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&R->stats[1], (unsigned long long)n);
    uint32_t *qc = &R->qcount[bounce * Q_PER_BOUNCE];
    uint32_t *qc_next = &R->qcount[(bounce + 1) * Q_PER_BOUNCE + Q_PATH];
    uint32_t *q_next = R->q_path[(bounce + 1) & 1];
    const int outside = R->has_medium ? 0 : -1;
    uint32_t i;
    while (warp_fetch(work, n, &i)) {
        const bool active = i < n;
        bool cont = false, cross = false;
        int family = -1;
        uint32_t pend = 0, slot = 0;
        if (active) {
            slot = queue[i];
            PathRec &P = R->path[slot];
            const PathVertex v = load_vertex(P);
            float betaW;
            Spec beta = ld_spec(P.beta, R->s_beta, slot, &betaW);
            const int med = R->cur_med[slot];
            const uint32_t ti = P.hit;
            uint32_t mflags;
            const float tHit = hit_distance(R, P, ti, v.ro, v.rd, &mflags);
            const int bm = boundary_medium(R, ti);
            SobolStream st = sobol_stream(P.sobol, v.meta);
            const SamplerParams &sp = R->sampler;
            // every boundary crossed inside a medium spends two dimensions, so a path can run past the host's tables (the
            // reference aborts there, sobol.cpp / lowdiscrepancy.h:229); such a path ends here and is counted
            bool alive = true;
            if (st.dim + 10 > sp.n_dims) {
                alive = false;
                atomicAdd(R->dim_overflows, 1ull);
            }
            bool sampledMedium = false;
            float t = tHit;
            if (alive && med >= 0) {  // ray.medium->Sample (homogeneous.cpp:49-76)
                const float uChannel = get1d(sp, st), uDist = get1d(sp, st);
                t = sample_medium_rgb(media_sigma_t(R, med), media_sigma_s(R, med), v.rd, tHit, uChannel, uDist, &beta, &sampledMedium);
            }
            if (alive && !is_black(beta)) {
                if (!sampledMedium) {
                    if (bm >= 0) {
                        // a medium boundary: nothing is emitted or scattered there; volpath.cpp:112 ends the path at maxDepth
                        if (v.bounces < R->max_depth) {
                            const DevSphere *bs = R->scene.spheres + (ti & SPHERE_HIT_MASK);
                            float th;
                            Isect is;
                            if (sphere_intersect(*bs, v.ro, v.rd, pt_inf(), &th, &is)) {
                                R->cur_med[slot] = dot(v.rd, is.n) > 0 ? outside : bm;          // GetMedium(ray.d)
                                const V3 no = offset_ray_origin(is.p, is.pError, is.n, v.rd);  // isect.SpawnRay(ray.d)
                                P.o = f4(no, v.etaScale);
                                P.d = f4(v.rd, __uint_as_float(meta_with_dim(v.meta, st.dim)));
                                st_spec(P.beta, R->s_beta, slot, beta, betaW);
                                cross = true;
                            }
                        }
                    } else {
                        // on to the surface vertex (or out of the scene)
                        st_spec(P.beta, R->s_beta, slot, beta, betaW);
                        P.d = f4(v.rd, __uint_as_float(meta_with_dim(v.meta, st.dim)));
                        if (ti != B200PT_MISS) family = hit_family(R->scene.materials, mflags);
                    }
                } else if (v.bounces < R->max_depth) {  // volpath.cpp:84-85
                    const Isect mi = medium_interaction(v.ro, v.rd, t);
                    if (R->n_lights > 0) {
                        float pickPdf;
                        const int lightNum = pick_light(R, mi.p, get1d(sp, st), &pickPdf);
                        if (pickPdf != 0) {
                            float uLight[2], uScattering[2];
                            get2d(sp, st, uLight);
                            get2d(sp, st, uScattering);
                            DirectOut dout;
                            Bsdf none;
                            none.n = 0;
                            estimate_direct<true>(R, mi, none, uScattering, lightNum, uLight, &dout, true, med);
                            pend = dout.pend;
                            if (pend) {
                                st_beta_ld(R->direct[slot], R->s_beta_ld, slot, beta, pickPdf);
                                R->direct[slot].sh_o = f4(dout.sh_o, __uint_as_float((uint32_t)lightNum));
                                if (pend & PEND_LIGHT) st_spec(R->direct[slot].A, R->s_A, slot, dout.A, dout.wA);
                                if (pend & PEND_BSDF) {
                                    R->direct[slot].mi_o = f4(dout.mi_o, dout.pdfB);
                                    R->direct[slot].mi_d = f4(dout.mi_d, 0.f);
                                    st_spec(R->direct[slot].B, R->s_B, slot, dout.B, dout.wB);
                                }
                                store_direct_general(R, slot, dout, med);
                            }
                            R->direct[slot].sh_d = f4(dout.sh_d, __uint_as_float(pend));
                        }
                    }
                    V3 wi;
                    float u2[2];
                    get2d(sp, st, u2);
                    hg_sample_p(R->media_g[med], mi.wo, &wi, u2);
                    const V3 no = offset_ray_origin(mi.p, mi.pError, mi.n, wi);
                    cont = true;
                    const float rrMax = max_comp(beta * v.etaScale);  // volpath.cpp:176-184
                    if (rrMax < R->rr_threshold && v.bounces > 3) cont = russian_roulette(rrMax, get1d(sp, st), &beta);
                    if (cont) {
                        P.o = f4(no, v.etaScale);
                        P.d = f4(wi, __uint_as_float(pack_meta(st.dim, v.bounces + 1, false)));
                        st_spec(P.beta, R->s_beta, slot, beta, 0.f);
                    }
                }
            }
        }
        append_family(R->q_mat, &qc[Q_MAT0], family, slot);
        append_vertex_out(R, qc, qc_next, q_next, pend, cont, slot);
        const uint32_t pc = warp_append(cross_count, cross);
        if (cross) q_cross[pc] = slot;
    }
}

// One segment of the direct-lighting rays' walk through the boundaries, after the segment's closest-hit launch.
// SHADOW: VisibilityTester::Tr (light.cpp:63-81) -- an opaque hit ends the ray occluded; otherwise the transmittance of
// the segment's medium is multiplied in and the ray is re-aimed at the light sample from behind the boundary
// (SpawnRayTo, interaction.h:73-78), or it arrived: A = f * (Li * Tr) * weight / lightPdf (integrator.cpp:141-158).
// !SHADOW: Scene::IntersectTr (scene.cpp:57-70) for the BSDF-sampled ray -- same direction behind a boundary; the walk
// ends on the first opaque hit: B = f * Le * Tr * weight / scatteringPdf if that is the sampled light (integrator.cpp:192-212).
template <bool SHADOW>
__global__ void __launch_bounds__(128, 4) k_direct_walk(const RenderDev *R, const uint32_t *queue, const uint32_t *count, uint32_t *q_out,
                                                        uint32_t *out_count, uint32_t *work, int count_rays) {
    const uint32_t n = *count;
    if (count_rays && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&R->stats[1], (unsigned long long)n);
    const int outside = R->has_medium ? 0 : -1;
    uint32_t i;
    while (warp_fetch(work, n, &i)) {
        bool again = false;
        uint32_t slot = 0;
        if (i < n) {
            slot = queue[i];
            if (SHADOW) {
                const float4 o4 = R->direct[slot].sh_o, d4 = R->direct[slot].sh_d, tr4 = R->sh_tr[slot];
                const V3 o = v3(o4), d = v3(d4);
                int m = (int)__float_as_uint(tr4.w);
                Spec Tr = rgb(tr4.x, tr4.y, tr4.z);
                const uint32_t ti = R->sh_hit[slot];
                const int bm = boundary_medium(R, ti);
                if (ti != B200PT_MISS && bm < 0) {
                    R->direct[slot].occluded = 1;  // an opaque surface between the point and the light
                } else {
                    float th = PT_SHADOW_TMAX;
                    Isect ii;
                    bool crossed = false;
                    if (ti != B200PT_MISS) crossed = sphere_intersect(R->scene.spheres[ti & SPHERE_HIT_MASK], o, d, PT_SHADOW_TMAX, &th, &ii);
                    if (!crossed) th = PT_SHADOW_TMAX;
                    if (m >= 0) Tr = Tr * medium_tr(media_sigma_t(R, m), d, th);
                    if (!crossed) {
                        float wA;
                        const Spec f = ld_spec(R->direct[slot].A, R->s_A, slot, &wA);
                        const float4 l4 = R->A2[slot];
                        const Spec Li = rgb(l4.x, l4.y, l4.z) * Tr;
                        const Spec A = wA < 0.f ? f * Li / 1.f : f * Li * wA / l4.w;
                        st_spec(R->direct[slot].A, R->s_A, slot, A, 0.f);
                        R->direct[slot].occluded = 0;
                    } else {
                        const V3 p1 = v3(R->sh_p1[slot]), p1e = v3(R->sh_p1e[slot]), p1n = v3(R->sh_p1n[slot]);
                        const V3 o2 = offset_ray_origin(ii.p, ii.pError, ii.n, p1 - ii.p);
                        const V3 target = offset_ray_origin(p1, p1e, p1n, o2 - p1);
                        const V3 d2 = target - o2;
                        m = dot(d2, ii.n) > 0 ? outside : bm;  // GetMedium(d)
                        R->direct[slot].sh_o = f4(o2, o4.w);
                        R->direct[slot].sh_d = f4(d2, d4.w);
                        R->sh_tr[slot] = make_float4(Tr.c[0], Tr.c[1], Tr.c[2], __uint_as_float((uint32_t)m));
                        again = true;
                    }
                }
            } else {
                const float4 o4 = R->direct[slot].mi_o, d4 = R->direct[slot].mi_d, tr4 = R->mi_tr[slot];
                const V3 o = v3(o4), wi = v3(d4);
                int m = (int)__float_as_uint(tr4.w);
                Spec Tr = rgb(tr4.x, tr4.y, tr4.z);
                const uint32_t ti = R->direct[slot].mis_hit;
                const int bm = boundary_medium(R, ti);
                float th = pt_inf();
                Isect ii;
                if (bm >= 0 && sphere_intersect(R->scene.spheres[ti & SPHERE_HIT_MASK], o, wi, pt_inf(), &th, &ii)) {
                    if (m >= 0) Tr = Tr * medium_tr(media_sigma_t(R, m), wi, th);
                    const V3 o2 = offset_ray_origin(ii.p, ii.pError, ii.n, wi);  // isect->SpawnRay(ray.d)
                    m = dot(wi, ii.n) > 0 ? outside : bm;
                    R->direct[slot].mi_o = f4(o2, o4.w);
                    R->mi_tr[slot] = make_float4(Tr.c[0], Tr.c[1], Tr.c[2], __uint_as_float((uint32_t)m));
                    again = true;
                } else {
                    const int lightNum = (int)__float_as_uint(R->direct[slot].sh_o.w);
                    const DevLight light = R->lights[lightNum];
                    Spec B = rgb1(0.f);
                    if (ti != B200PT_MISS && ti == light.tri) {
                        // distance and normal of the light's shape as this segment meets it
                        float t = pt_inf();
                        V3 ln = mk(0.f, 0.f, 0.f);
                        if (is_sphere_hit(ti)) {
                            Isect li;
                            if (sphere_intersect(R->scene.spheres[ti & SPHERE_HIT_MASK], o, wi, pt_inf(), &t, &li)) ln = li.n;
                        } else {
                            const F4 *tp = R->scene.tris + (size_t)ti * 3;
                            const F4 t0 = ld_f4(tp), t1 = ld_f4(tp + 1), t2 = ld_f4(tp + 2);
                            const uint32_t lflags = __float_as_uint(t1.w);
                            TriHit h;
                            if (triangle_test(v3(t0), v3(t1), v3(t2), o, make_shear(wi), pt_inf(), &h)) {
                                TriShading lsh;
                                load_shading<true>(R->scene, ti, lflags, &lsh);
                                Isect li;
                                fill_isect(v3(t0), v3(t1), v3(t2), (lflags & B200PT_TRI_FLIP) != 0, lsh, h, wi, &li);
                                ln = li.n;
                                t = h.t;
                            }
                        }
                        if (m >= 0) Tr = Tr * medium_tr(media_sigma_t(R, m), wi, t);
                        const Spec Le = (light.two_sided || dot(ln, -wi) > 0) ? light_emit(R, lightNum, light) : rgb1(0.f);
                        if (!is_black(Le)) {
                            float wB;
                            const Spec f = ld_spec(R->direct[slot].B, R->s_B, slot, &wB);
                            B = f * Le * Tr * wB / o4.w;
                        }
                    }
                    st_spec(R->direct[slot].B, R->s_B, slot, B, 0.f);
                }
            }
        }
        const uint32_t pos = warp_append(out_count, again);
        if (again) q_out[pos] = slot;
    }
}
#endif  // B200PT_MEDIA_GENERAL

// L += beta * (EstimateDirect(...) / lightPdf)   (path.cpp:122-127, integrator.cpp:104-105)
__global__ void __launch_bounds__(256) k_resolve(const RenderDev *R, int bounce, uint32_t *work) {
    const uint32_t n = R->qcount[bounce * Q_PER_BOUNCE + Q_PATH];
    const uint32_t *queue = R->q_path[bounce & 1];
    uint32_t i;
    while (warp_fetch(work, n, &i)) {
        if (i >= n) continue;
        const uint32_t slot = queue[i];
        DirectRec &D = R->direct[slot];
        const float4 sd = D.sh_d;
        const uint32_t pend = __float_as_uint(sd.w);
        if (!pend) continue;
#if B200PT_NSPEC == 3
        Spec Ld = rgb1(0.f);
        bool any = false;
        if ((pend & PEND_LIGHT) && !D.occluded) {
            float w_;
            Ld = Ld + ld_spec(D.A, R->s_A, slot, &w_);
            any = true;
        }
        if (pend & PEND_BSDF) {
            const uint32_t lightNum = __float_as_uint(D.sh_o.w);
            float w_;
            const Spec B = ld_spec(D.B, R->s_B, slot, &w_);
            if (D.mis_hit == R->lights[lightNum].tri && !is_black(B)) {
                Ld = Ld + B;
                any = true;
            }
        }
        if (any) {
            float pickPdf, LW;
            const Spec betaLd = ld_spec(D.beta_ld, R->s_beta_ld, slot, &pickPdf);
            PathRec &P = R->path[slot];
            const Spec L = ld_spec(P.L, R->s_L, slot, &LW) + betaLd * (Ld / pickPdf);
            st_spec(P.L, R->s_L, slot, L, LW);
        }
#else
        // 60 bins: streamed through the slot's rows, bin by bin (Ld = 0 + A + B; L += beta_ld * (Ld / pickPdf))
        const bool takeA = (pend & PEND_LIGHT) && !D.occluded;
        bool takeB = false;
        if (pend & PEND_BSDF) {
            const uint32_t lightNum = __float_as_uint(D.sh_o.w);
            if (D.mis_hit == R->lights[lightNum].tri) {
                const float *sB = R->s_B + (size_t)slot * B200PT_NSPEC;
                for (int b = 0; b < B200PT_NSPEC && !takeB; ++b) takeB = sB[b] != 0.f;
            }
        }
        if (takeA || takeB) {
            const float pickPdf = D.beta_ld.w;
            const float4 *sA = reinterpret_cast<const float4 *>(R->s_A + (size_t)slot * B200PT_NSPEC);
            const float4 *sB = reinterpret_cast<const float4 *>(R->s_B + (size_t)slot * B200PT_NSPEC);
            const float4 *sBl = reinterpret_cast<const float4 *>(R->s_beta_ld + (size_t)slot * B200PT_NSPEC);
            float4 *sL = reinterpret_cast<float4 *>(R->s_L + (size_t)slot * B200PT_NSPEC);
#pragma unroll 3
            for (int q = 0; q < B200PT_NSPEC / 4; ++q) {
                float4 Ld = make_float4(0.f, 0.f, 0.f, 0.f);
                if (takeA) {
                    const float4 a = sA[q];
                    Ld = make_float4(Ld.x + a.x, Ld.y + a.y, Ld.z + a.z, Ld.w + a.w);
                }
                if (takeB) {
                    const float4 b = sB[q];
                    Ld = make_float4(Ld.x + b.x, Ld.y + b.y, Ld.z + b.z, Ld.w + b.w);
                }
                const float4 l = sL[q], bl = sBl[q];
                sL[q] = make_float4(l.x + bl.x * (Ld.x / pickPdf), l.y + bl.y * (Ld.y / pickPdf), l.z + bl.z * (Ld.z / pickPdf),
                                    l.w + bl.w * (Ld.w / pickPdf));
            }
        }
#endif
        D.sh_d = make_float4(sd.x, sd.y, sd.z, 0.f);
    }
}

#if B200PT_NSPEC == 3
// path.cpp:89-100 for a path ray of `bounce` that found no intersection: at the first vertex or after a specular bounce,
// L += beta * Le(ray) for each infinite light in Scene::infiniteLights order.  The path ends there (path.cpp:103).
__global__ void __launch_bounds__(256) k_escape(const RenderDev *R, int bounce, uint32_t *work) {
    const uint32_t n = R->qcount[bounce * Q_PER_BOUNCE + Q_PATH];
    const uint32_t *queue = R->q_path[bounce & 1];
    uint32_t i;
    while (warp_fetch(work, n, &i)) {
        if (i >= n) continue;
        const uint32_t slot = queue[i];
        PathRec &P = R->path[slot];
        if (P.hit != B200PT_MISS) continue;
        const PathVertex v = load_vertex(P);
        if (!(v.bounces == 0 || v.specularBounce)) continue;
        float betaW, LW;
        const Spec beta = ld_spec(P.beta, R->s_beta, slot, &betaW);
        Spec L = ld_spec(P.L, R->s_L, slot, &LW);
        for (int k = 0; k < R->n_infinite; ++k) L = L + beta * infinite_le(R->infinite[k], v.rd);
        st_spec(P.L, R->s_L, slot, L, LW);
    }
}

// SpatialLightDistribution::ComputeDistribution's terms of the infinite lights (lightdistrib.cpp:256-275): Li.y() / pdf of
// Sample_Li at the voxel's 128 Halton points.  Runs after k_spatial_contrib and replaces those lights' entries.
__global__ void __launch_bounds__(128) k_spatial_infinite(const RenderDev *R) {
    const SpatialGrid &g = R->grid;
    const long long nvox = (long long)g.nv[0] * g.nv[1] * g.nv[2];
    const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= nvox * R->n_lights) return;
    const int j = (int)(id % R->n_lights);
    const DevLight &light = R->lights[j];
    if (light.kind != B200PT_LIGHT_INFINITE) return;
    const DevInfinite &L = R->infinite[light.two_sided];
    const long long vox = id / R->n_lights;
    const int pi[3] = {(int)(vox % g.nv[0]), (int)((vox / g.nv[0]) % g.nv[1]), (int)(vox / ((long long)g.nv[0] * g.nv[1]))};
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
        V3 wi, pT;
        float pdf;
        const Spec Li = infinite_sample_li(L, po, u, &wi, &pdf, &pT);
        if (pdf > 0) contrib += lum(Li) / pdf;
    }
    R->sp_func[vox * R->n_lights + j] = contrib;
}
#endif

#if B200PT_NSPEC == 3  // spectrum-independent: compiled once, in the RGBSpectrum translation unit
// Sobol' byte tables: table[dim][k][b] = XOR of SobolMatrices32[dim*52 + 8k + i] over the set bits i of b.
__global__ void k_sobol_table(const uint32_t *mat32, uint32_t *table, int n_dims) {
    const int id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= n_dims * 5 * 256) return;
    const int b = id & 255, k = (id >> 8) % 5, dim = id / (5 * 256);
    uint32_t v = 0;
    for (int i = 0; i < 8; ++i)
        if (((b >> i) & 1) && 8 * k + i < 52) v ^= mat32[dim * 52 + 8 * k + i];
    table[id] = v;
}
void launch_sobol_table(const uint32_t *mat32, uint32_t *table, int n_dims, cudaStream_t s) {
    const int n = n_dims * 5 * 256;
    B200PT_LAUNCH(B200PT_KERNEL(k_sobol_table), (n + 255) / 256, 256, s, mat32, table, n_dims);
}

#endif  // B200PT_NSPEC == 3
// --------------------------------------------------- spatial light distribution
// SpatialLightDistribution::ComputeDistribution for every voxel (the reference fills its hash table
// lazily; a voxel's distribution is a pure function of the voxel).  One thread per (voxel, light)
// accumulates the 128 Halton terms in order, then one thread per voxel builds the Distribution1D.
__global__ void __launch_bounds__(128) k_spatial_contrib(const RenderDev *R) {
    const SpatialGrid &g = R->grid;
    const long long nvox = (long long)g.nv[0] * g.nv[1] * g.nv[2];
    const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= nvox * R->n_lights) return;
    const int j = (int)(id % R->n_lights);
    const long long vox = id / R->n_lights;
    const int vx = (int)(vox % g.nv[0]), vy = (int)((vox / g.nv[0]) % g.nv[1]), vz = (int)(vox / ((long long)g.nv[0] * g.nv[1]));
    const DevLight light = R->lights[j];
    const bool isDelta = light.kind != 0;
    const Spec lemit = light_emit(R, j, light);
    DeltaLight dl;
    if (isDelta) dl = delta_of(R->lights[j], lemit);
    const bool onSphere = !isDelta && is_sphere_hit(light.tri);
    const F4 *tp = R->scene.tris + (size_t)((onSphere || isDelta) ? 0u : light.tri) * 3;
    F4 t0 = {0.f, 0.f, 0.f, 0.f}, t1 = t0, t2 = t0;
    if (!onSphere && !isDelta) {
        t0 = ld_f4(tp);
        t1 = ld_f4(tp + 1);
        t2 = ld_f4(tp + 2);
    }
    const uint32_t lflags = __float_as_uint(t1.w);
    TriShading lsh;
    load_shading<true>(R->scene, isDelta ? 0u : light.tri, lflags, &lsh);
    R->sp_func[vox * R->n_lights + j] =
        spatial_light_contrib(g, vx, vy, vz, v3(t0), v3(t1), v3(t2), (lflags & B200PT_TRI_FLIP) != 0, lsh, lemit,
                              light.two_sided != 0, onSphere ? R->scene.spheres + (light.tri & SPHERE_HIT_MASK) : nullptr,
                              isDelta ? &dl : nullptr);
}
__global__ void __launch_bounds__(128) k_spatial_cdf(const RenderDev *R) {
    const SpatialGrid &g = R->grid;
    const long long nvox = (long long)g.nv[0] * g.nv[1] * g.nv[2];
    const long long vox = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vox >= nvox) return;
    const int n = R->n_lights;
    float *func = R->sp_func + vox * n, *cdf = R->sp_cdf + vox * (n + 1);
    // lightdistrib.cpp:277-299
    float sumContrib = 0.f;
    for (int i = 0; i < n; ++i) sumContrib = sumContrib + func[i];
    const float avgContrib = sumContrib / (float)(128ull * (unsigned long long)n);
    const float minContrib = (avgContrib > 0) ? (float)(.001 * (double)avgContrib) : 1.f;
    for (int i = 0; i < n; ++i) func[i] = pt_max(func[i], minContrib);
    // Distribution1D, sampling.h:57-71
    cdf[0] = 0;
    for (int i = 1; i < n + 1; ++i) cdf[i] = cdf[i - 1] + func[i - 1] / n;
    const float funcInt = cdf[n];
    if (funcInt == 0) {
        for (int i = 1; i < n + 1; ++i) cdf[i] = (float)i / (float)n;
    } else {
        for (int i = 1; i < n + 1; ++i) cdf[i] /= funcInt;
    }
    R->sp_func_int[vox] = funcInt;
}

// ------------------------------------------------------------------------ film
// One block per tile, one thread per pixel of the tile's FilmTile (the tile
// plus a one-pixel apron, film.cpp:95-106).  A thread re-creates the
// reference's accumulation order for its pixel: source pixels in row-major
// order within the tile, samples in order (integrator.cpp:263-325), each
// sample added to every pixel of its box-filter footprint (film.h:121-161),
// then one RGB->XYZ conversion and add into the film (film.cpp:117-130).
__global__ void __launch_bounds__(18 * 18) k_film(const RenderDev *R, uint32_t first_tile) {
    const uint32_t tb = blockIdx.x;
    const int tile = R->tile_list[first_tile + tb];
    const TileRect t = tile_rect(R, tile);
    const int X = t.x0 - 1 + (int)threadIdx.x, Y = t.y0 - 1 + (int)threadIdx.y;
    // FilmTile pixel bounds: [x0-1, x1+1) x [y0-1, y1+1) clipped to the cropped film
    if (X >= t.x1 + 1 || Y >= t.y1 + 1) return;
    if (X < R->crop[0] || X >= R->crop[2] || Y < R->crop[1] || Y >= R->crop[3]) return;
    const uint32_t spp = (uint32_t)R->sampler.spp;
    const float maxLum = R->max_sample_luminance;
    Spec sum = rgb1(0.f);
    float wsum = 0.f;
    for (int sy = Y - 1; sy <= Y + 1; ++sy)
        for (int sx = X - 1; sx <= X + 1; ++sx) {
            if (!pixel_rendered(R, t, sx, sy)) continue;
            const uint32_t pix = (uint32_t)((sy - t.y0) * 16 + (sx - t.x0));
            const bool own = (sx == X && sy == Y);
            if (!own && !R->pix_bleed[tb * 256u + pix]) continue;
            const uint32_t base = (tb * 256u + pix) * spp;
            for (uint32_t s = 0; s < spp; ++s) {
                float vw;
                Spec Lv = ld_spec(R->path[base + s].L, R->s_L, base + s, &vw);
                if (!own) {
                    const uint32_t code = __float_as_uint(vw);
                    const bool cx = (X == sx) || (X == sx - 1 && (code & 1u)) || (X == sx + 1 && (code & 2u));
                    const bool cy = (Y == sy) || (Y == sy - 1 && (code & 4u)) || (Y == sy + 1 && (code & 8u));
                    if (!(cx && cy)) continue;
                }
                // integrator.cpp:294-315
                if (has_nans(Lv))
                    Lv = rgb1(0.f);
                else if (lum(Lv) < -1e-5f)
                    Lv = rgb1(0.f);
                else if (pt_isinf(lum(Lv)))
                    Lv = rgb1(0.f);
                if (lum(Lv) > maxLum) Lv = Lv * (maxLum / lum(Lv));  // film.h:124-125
                sum = sum + Lv * 1.f * 1.f;                           // L * sampleWeight * filterWeight
                wsum += 1.f;
            }
        }
    if (wsum != 0.f) {
        float xyz[3];
        rgb_to_xyz(sum, xyz);
        float *fp = reinterpret_cast<float *>(R->film + (size_t)(Y - R->crop[1]) * (R->crop[2] - R->crop[0]) +
                                              (X - R->crop[0]));
        atomicAdd(fp + 0, xyz[0]);
        atomicAdd(fp + 1, xyz[1]);
        atomicAdd(fp + 2, xyz[2]);
        atomicAdd(fp + 3, wsum);
    }
}

// ---- general pixel filter -------------------------------------------------------------------------------------
// FilmTile pixel bounds of a tile (Film::GetFilmTile, film.cpp:95-106)
struct TileFilm {
    int bx0, by0, bx1, by1;
};
__device__ __forceinline__ TileFilm tile_film_bounds(const RenderDev *R, const TileRect &t) {
    TileFilm f;
    f.bx0 = max((int)ceilf((float)t.x0 - 0.5f - R->filter_radius[0]), R->crop[0]);
    f.by0 = max((int)ceilf((float)t.y0 - 0.5f - R->filter_radius[1]), R->crop[1]);
    f.bx1 = min((int)floorf((float)t.x1 - 0.5f + R->filter_radius[0]) + 1, R->crop[2]);
    f.by1 = min((int)floorf((float)t.y1 - 0.5f + R->filter_radius[1]) + 1, R->crop[3]);
    return f;
}
// One block per tile, one thread per FilmTile pixel: the thread replays FilmTile::AddSample (film.h:121-161) for its
// pixel over the tile's samples in the reference's order (pixels row-major, samples in order) and stores what
// MergeFilmTile would add to the film (film.cpp:117-130).
__global__ void __launch_bounds__(1024) k_film_tile(const RenderDev *R, uint32_t first_tile) {
    const uint32_t tb = blockIdx.x;
    const int tile = R->tile_list[first_tile + tb];
    const TileRect t = tile_rect(R, tile);
    const TileFilm f = tile_film_bounds(R, t);
    const int fw = 16 + 2 * R->apron[0], fh = 16 + 2 * R->apron[1];
    const int lx = (int)threadIdx.x, ly = (int)threadIdx.y;
    // local (lx, ly) <-> pixel: the tile's unclipped FilmTile window starts at (x0 - apron, y0 - apron)
    const int X = t.x0 - R->apron[0] + lx, Y = t.y0 - R->apron[1] + ly;
    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
    if (X >= f.bx0 && X < f.bx1 && Y >= f.by0 && Y < f.by1) {
        const uint32_t spp = (uint32_t)R->sampler.spp;
        const float maxLum = R->max_sample_luminance;
        const float rx = R->filter_radius[0], ry = R->filter_radius[1];
        Spec sum = rgb1(0.f);
        float wsum = 0.f;
        // source pixels whose samples can reach this pixel: |pFilm - 0.5 - X| <= r with pFilm in [sx, sx + 1)
        const int sx0 = max(t.x0, (int)ceilf((float)X - 0.5f - rx) - 1), sx1 = min(t.x1 - 1, (int)floorf((float)X + 0.5f + rx) + 1);
        const int sy0 = max(t.y0, (int)ceilf((float)Y - 0.5f - ry) - 1), sy1 = min(t.y1 - 1, (int)floorf((float)Y + 0.5f + ry) + 1);
        for (int sy = sy0; sy <= sy1; ++sy)
            for (int sx = sx0; sx <= sx1; ++sx) {
                if (!pixel_rendered(R, t, sx, sy)) continue;
                const uint32_t pix = (uint32_t)((sy - t.y0) * 16 + (sx - t.x0));
                const size_t base = ((size_t)tb * 256u + pix) * spp;
                for (uint32_t s = 0; s < spp; ++s) {
                    const float2 pf = R->pfilm[base + s];
                    const float dx = pf.x - 0.5f, dy = pf.y - 0.5f;
                    const int q0x = max((int)ceilf(dx - rx), f.bx0), q1x = min((int)floorf(dx + rx) + 1, f.bx1);
                    const int q0y = max((int)ceilf(dy - ry), f.by0), q1y = min((int)floorf(dy + ry) + 1, f.by1);
                    if (X < q0x || X >= q1x || Y < q0y || Y >= q1y) continue;
                    const float fx = fabsf(((float)X - dx) * R->filter_inv_radius[0] * 16.f);
                    const float fy = fabsf(((float)Y - dy) * R->filter_inv_radius[1] * 16.f);
                    const int ifx = min((int)floorf(fx), 15), ify = min((int)floorf(fy), 15);
                    const float w = R->filter_table[ify * 16 + ifx];
                    float vw;
                    Spec Lv = ld_spec(R->path[(uint32_t)(base + s)].L, R->s_L, (uint32_t)(base + s), &vw);
                    // integrator.cpp:294-315
                    if (has_nans(Lv))
                        Lv = rgb1(0.f);
                    else if (lum(Lv) < -1e-5f)
                        Lv = rgb1(0.f);
                    else if (pt_isinf(lum(Lv)))
                        Lv = rgb1(0.f);
                    if (lum(Lv) > maxLum) Lv = Lv * (maxLum / lum(Lv));  // film.h:124-125
                    sum = sum + Lv * 1.f * w;                             // L * sampleWeight * filterWeight
                    wsum += w;
                }
            }
        float xyz[3];
        rgb_to_xyz(sum, xyz);
        out = make_float4(xyz[0], xyz[1], xyz[2], wsum);
    }
    if (lx < fw && ly < fh) R->tile_film[((size_t)tb * fh + ly) * fw + lx] = out;
}
__global__ void k_film_tile_slots(const RenderDev *R, uint32_t first_tile, uint32_t n_batch_tiles) {
    const uint32_t tb = blockIdx.x * blockDim.x + threadIdx.x;
    if (tb < n_batch_tiles) R->tile_slot[R->tile_list[first_tile + tb]] = (int32_t)tb;
}
// One thread per film pixel: adds the FilmTile values of the batch's tiles that cover it, in ascending tile order.
__global__ void k_film_merge(const RenderDev *R) {
    const int w = R->crop[2] - R->crop[0], h = R->crop[3] - R->crop[1];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * h) return;
    const int X = R->crop[0] + i % w, Y = R->crop[1] + i / w;
    const int fw = 16 + 2 * R->apron[0], fh = 16 + 2 * R->apron[1];
    const int tx0 = max(0, (X - R->apron[0] - R->sampler.sb[0]) >> 4), tx1 = min(R->tiles_x - 1, (X + R->apron[0] - R->sampler.sb[0]) >> 4);
    const int ty0 = max(0, (Y - R->apron[1] - R->sampler.sb[1]) >> 4), ty1 = min(R->tiles_y - 1, (Y + R->apron[1] - R->sampler.sb[1]) >> 4);
    float4 acc = R->film[i];
    bool touched = false;
    for (int ty = ty0; ty <= ty1; ++ty)
        for (int tx = tx0; tx <= tx1; ++tx) {
            const int tile = ty * R->tiles_x + tx;
            const int32_t tb = R->tile_slot[tile];
            if (tb < 0) continue;
            const TileRect t = tile_rect(R, tile);
            const TileFilm f = tile_film_bounds(R, t);
            if (X < f.bx0 || X >= f.bx1 || Y < f.by0 || Y >= f.by1) continue;
            const int lx = X - (t.x0 - R->apron[0]), ly = Y - (t.y0 - R->apron[1]);
            const float4 v = R->tile_film[((size_t)tb * fh + ly) * fw + lx];
            acc.x += v.x;
            acc.y += v.y;
            acc.z += v.z;
            acc.w += v.w;
            touched = true;
        }
    if (touched) R->film[i] = acc;
}
__global__ void k_film_tile_slots_reset(const RenderDev *R, uint32_t first_tile, uint32_t n_batch_tiles) {
    const uint32_t tb = blockIdx.x * blockDim.x + threadIdx.x;
    if (tb < n_batch_tiles) R->tile_slot[R->tile_list[first_tile + tb]] = -1;
}

#if B200PT_NSPEC == 3  // spectrum-independent: compiled once, in the RGBSpectrum translation unit
__global__ void k_accumulate_stats(const RenderDev *R) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    unsigned long long regular = 0, shadow = 0;
    for (int b = 0; b <= R->max_depth; ++b) {
        regular += R->qcount[b * Q_PER_BOUNCE + Q_PATH] + R->qcount[b * Q_PER_BOUNCE + Q_MIS];
        shadow += R->qcount[b * Q_PER_BOUNCE + Q_SHADOW];
    }
    if (R->volpath) {
        // VolPathIntegrator's direct-lighting rays go through VisibilityTester::Tr -> Scene::Intersect (light.cpp:63-81):
        // the reference counts them as regular intersection tests, its shadow-ray counter stays 0
        regular += shadow;
        shadow = 0;
    }
    R->stats[0] += R->qcount[Q_PATH];
    R->stats[1] += regular;
    R->stats[2] += shadow;
}

// Film::WriteImage pixel pipeline (film.cpp:174-203); splats are always zero here.
__global__ void k_film_rgb(const float4 *film, float *out, int n, float scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = film[i];
    float xyz[3] = {p.x, p.y, p.z}, c[3];
    xyz_to_rgb(xyz, c);
    if (p.w != 0) {
        const float invWt = 1.0f / p.w;
        c[0] = pt_max(0.f, c[0] * invWt);
        c[1] = pt_max(0.f, c[1] * invWt);
        c[2] = pt_max(0.f, c[2] * invWt);
    }
    float zero[3] = {0.f, 0.f, 0.f}, splat[3];
    xyz_to_rgb(zero, splat);
    for (int k = 0; k < 3; ++k) {
        c[k] += 1.f * splat[k];
        c[k] *= scale;
        out[3 * i + k] = c[k];
    }
}

__global__ void k_debug_sobol(const RenderDev *R, int px, int py, long long sample, int dim0, int n, float *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const SamplerParams &sp = R->sampler;
    const uint64_t idx = sampler_index(sp, (uint64_t)sample, px, py);
    out[i] = sampler_sample(sp, idx, dim0 + i, px, py);
}

__global__ void k_debug_camera(const RenderDev *R, int px, int py, int n, b200pt_ray *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const SamplerParams &sp = R->sampler;
    SobolStream st;
    st.index = sampler_index(sp, (uint64_t)i, px, py);
    st.dim = 0;
    st.px = px;
    st.py = py;
    float u[2], ul[2];
    get2d(sp, st, u);
    float pFilm[2] = {(float)px + u[0], (float)py + u[1]};
    (void)get1d(sp, st);
    get2d(sp, st, ul);
    V3 o, d;
    float tMax;
    generate_camera_ray(R->camera, pFilm, ul, &o, &d, &tMax);
    b200pt_ray r;
    r.o[0] = o.x;
    r.o[1] = o.y;
    r.o[2] = o.z;
    r.t_max = tMax;
    r.d[0] = d.x;
    r.d[1] = d.y;
    r.d[2] = d.z;
    r.pad = 0.f;
    out[i] = r;
}

#endif  // B200PT_NSPEC == 3
// -------------------------------------------------------------------- launchers
void launch_raygen(const RenderDev *dev, uint32_t batch_first_tile, uint32_t n_batch_tiles, uint32_t n_slots, bool keep_pfilm,
                   cudaStream_t s) {
    (void)n_batch_tiles;
#if B200PT_NSPEC == 3
    if (keep_pfilm) {
        B200PT_LAUNCH(B200PT_KERNEL(k_raygen_pfilm), (n_slots + 255) / 256, 256, s, dev, batch_first_tile, n_slots);
        return;
    }
#else
    (void)keep_pfilm;
#endif
    B200PT_LAUNCH(B200PT_KERNEL(k_raygen), (n_slots + 255) / 256, 256, s, dev, batch_first_tile, n_slots);
}

#if B200PT_NSPEC == 3  // spectrum-independent: compiled once, in the RGBSpectrum translation unit
template <class ALPHA>
static void launch_trace_as(const TraceArgs &a, bool any_hit, bool classify, bool count, int grid, cudaStream_t s) {
    if (any_hit) {
        if (count)
            B200PT_LAUNCH(B200PT_KERNEL(k_trace<true, false, true, ALPHA>), grid, 128, s, a);
        else
            B200PT_LAUNCH(B200PT_KERNEL(k_trace<true, false, false, ALPHA>), grid, 128, s, a);
    } else if (classify) {
        if (count)
            B200PT_LAUNCH(B200PT_KERNEL(k_trace<false, true, true, ALPHA>), grid, 128, s, a);
        else
            B200PT_LAUNCH(B200PT_KERNEL(k_trace<false, true, false, ALPHA>), grid, 128, s, a);
    } else {
        if (count)
            B200PT_LAUNCH(B200PT_KERNEL(k_trace<false, false, true, ALPHA>), grid, 128, s, a);
        else
            B200PT_LAUNCH(B200PT_KERNEL(k_trace<false, false, false, ALPHA>), grid, 128, s, a);
    }
}
void launch_trace(const TraceArgs &a, bool any_hit, bool classify, bool count, int n_sm, cudaStream_t s) {
#ifdef B200PT_HOST_EMU
    const int grid = n_sm;  // the per-ray k_trace of the check build has no occupancy to fill
#else
    const int grid = n_sm * B200PT_TRACE_CTAS;
#endif
    if (a.alpha_masks)
        launch_trace_as<AlphaTest>(a, any_hit, classify, count, grid, s);
    else
        launch_trace_as<NoAlpha>(a, any_hit, classify, count, grid, s);
}

#ifndef B200PT_HOST_EMU
template <class ALPHA>
static void launch_trace2_as(const TraceArgs &a, bool any_hit, bool classify, int grid, cudaStream_t s) {
    if (any_hit)
        B200PT_LAUNCH(B200PT_KERNEL(k_trace2<true, false, ALPHA>), grid, 128, s, a);
    else if (classify)
        B200PT_LAUNCH(B200PT_KERNEL(k_trace2<false, true, ALPHA>), grid, 128, s, a);
    else
        B200PT_LAUNCH(B200PT_KERNEL(k_trace2<false, false, ALPHA>), grid, 128, s, a);
}
void launch_trace2(const TraceArgs &a, bool any_hit, bool classify, int n_sm, cudaStream_t s) {
    if (a.alpha_masks)
        launch_trace2_as<AlphaTest>(a, any_hit, classify, n_sm * 6, s);
    else
        launch_trace2_as<NoAlpha>(a, any_hit, classify, n_sm * 6, s);
}
#endif

template <class ALPHA>
static void launch_spheres_as(const TraceArgs &a, bool any_hit, bool classify, int grid, cudaStream_t s) {
    if (any_hit)
        B200PT_LAUNCH(B200PT_KERNEL(k_spheres<true, false, ALPHA>), grid, 128, s, a);
    else if (classify)
        B200PT_LAUNCH(B200PT_KERNEL(k_spheres<false, true, ALPHA>), grid, 128, s, a);
    else
        B200PT_LAUNCH(B200PT_KERNEL(k_spheres<false, false, ALPHA>), grid, 128, s, a);
}
void launch_spheres(const TraceArgs &a, bool any_hit, bool classify, int grid, cudaStream_t s) {
    if (a.alpha_masks)
        launch_spheres_as<AlphaTest>(a, any_hit, classify, grid, s);
    else
        launch_spheres_as<NoAlpha>(a, any_hit, classify, grid, s);
}

#endif  // B200PT_NSPEC == 3
void launch_shade(const RenderDev *dev, int material, bool vertex_data, int bounce, uint32_t *work, int grid,
                  cudaStream_t s) {
#if B200PT_NSPEC == 3
#define B200PT_SHADE(M)                                                                         \
    case M:                                                                                     \
        if (vertex_data)                                                                        \
            B200PT_LAUNCH(B200PT_KERNEL(k_shade<M, true>), grid, 128, s, dev, bounce, work);    \
        else                                                                                    \
            B200PT_LAUNCH(B200PT_KERNEL(k_shade<M, false>), grid, 128, s, dev, bounce, work);   \
        break;
#else
    // the 60-bin build instantiates only the general variant (VTX = true handles every scene; the lean one is a
    // register-pressure optimisation of the RGB build): half the compile time of that translation unit
    (void)vertex_data;
#define B200PT_SHADE(M)                                                                      \
    case M:                                                                                  \
        B200PT_LAUNCH(B200PT_KERNEL(k_shade<M, true>), grid, 128, s, dev, bounce, work);     \
        break;
#endif
    switch (material) {
        B200PT_SHADE(B200PT_MAT_MATTE)
        B200PT_SHADE(B200PT_MAT_PLASTIC)
        B200PT_SHADE(B200PT_MAT_METAL)
        B200PT_SHADE(B200PT_MAT_GLASS)
    }
#undef B200PT_SHADE
}

void launch_resolve(const RenderDev *dev, int bounce, uint32_t *work, int grid, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_resolve), grid, 256, s, dev, bounce, work);
}
#if B200PT_NSPEC == 3
void launch_escape(const RenderDev *dev, int bounce, uint32_t *work, int grid, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_escape), grid, 256, s, dev, bounce, work);
}
#endif

void launch_medium(const RenderDev *dev, int bounce, uint32_t *work, int grid, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_medium), grid, 128, s, dev, bounce, work);
}
#if B200PT_MEDIA_GENERAL
void launch_medium_general(const RenderDev *dev, const RenderDev &host, int bounce, const uint32_t *queue, const uint32_t *count,
                           int out, uint32_t *cross_count, uint32_t *work, bool count_rays, int grid, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_medium_general), grid, 128, s, dev, bounce, queue, count, host.q_cross[out], cross_count, work,
                  count_rays ? 1 : 0);
}
void launch_direct_walk(const RenderDev *dev, const RenderDev &host, bool shadow, const uint32_t *queue, const uint32_t *count,
                        int out, uint32_t *walk_count, uint32_t *work, bool count_rays, int grid, cudaStream_t s) {
    if (shadow)
        B200PT_LAUNCH(B200PT_KERNEL(k_direct_walk<true>), grid, 128, s, dev, queue, count, host.q_walk[out], walk_count, work,
                      count_rays ? 1 : 0);
    else
        B200PT_LAUNCH(B200PT_KERNEL(k_direct_walk<false>), grid, 128, s, dev, queue, count, host.q_walk[out], walk_count, work,
                      count_rays ? 1 : 0);
}
#endif

void launch_spatial_build(const RenderDev *dev, const RenderDev &host, cudaStream_t s) {
    const long long nvox = (long long)host.grid.nv[0] * host.grid.nv[1] * host.grid.nv[2];
    const long long n1 = nvox * host.n_lights;
    B200PT_LAUNCH(B200PT_KERNEL(k_spatial_contrib), (unsigned)((n1 + 127) / 128), 128, s, dev);
#if B200PT_NSPEC == 3
    if (host.n_infinite > 0) B200PT_LAUNCH(B200PT_KERNEL(k_spatial_infinite), (unsigned)((n1 + 127) / 128), 128, s, dev);
#endif
    B200PT_LAUNCH(B200PT_KERNEL(k_spatial_cdf), (unsigned)((nvox + 127) / 128), 128, s, dev);
}

void launch_film(const RenderDev *dev, uint32_t batch_first_tile, uint32_t n_batch_tiles, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_film), n_batch_tiles, dim3(18, 18), s, dev, batch_first_tile);
}

void launch_film_general(const RenderDev *dev, const RenderDev &host, uint32_t batch_first_tile, uint32_t n_batch_tiles,
                         cudaStream_t s) {
    const dim3 block((unsigned)(16 + 2 * host.apron[0]), (unsigned)(16 + 2 * host.apron[1]));
    B200PT_LAUNCH(B200PT_KERNEL(k_film_tile_slots), (n_batch_tiles + 255) / 256, 256, s, dev, batch_first_tile, n_batch_tiles);
    B200PT_LAUNCH(B200PT_KERNEL(k_film_tile), n_batch_tiles, block, s, dev, batch_first_tile);
    const int npix = (host.crop[2] - host.crop[0]) * (host.crop[3] - host.crop[1]);
    B200PT_LAUNCH(B200PT_KERNEL(k_film_merge), (npix + 255) / 256, 256, s, dev);
    B200PT_LAUNCH(B200PT_KERNEL(k_film_tile_slots_reset), (n_batch_tiles + 255) / 256, 256, s, dev, batch_first_tile, n_batch_tiles);
}

#if B200PT_NSPEC == 3  // spectrum-independent: compiled once, in the RGBSpectrum translation unit
void launch_accumulate_stats(const RenderDev *dev, uint32_t, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_accumulate_stats), 1, 32, s, dev);
}

void launch_debug_sobol(const RenderDev *dev, int px, int py, long long sample, int dim0, int n, float *out,
                        cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_debug_sobol), (n + 63) / 64, 64, s, dev, px, py, sample, dim0, n, out);
}
void launch_debug_camera(const RenderDev *dev, int px, int py, int n, b200pt_ray *out, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_debug_camera), (n + 63) / 64, 64, s, dev, px, py, n, out);
}
void launch_film_rgb(const float4 *film, float *rgb, int n_pixels, float scale, cudaStream_t s) {
    B200PT_LAUNCH(B200PT_KERNEL(k_film_rgb), (n_pixels + 255) / 256, 256, s, film, rgb, n_pixels, scale);
}

#endif  // B200PT_NSPEC == 3
#if B200PT_NSPEC != 3
// SampledSpectrum::X / Y / Z of the host (b200pt_scene_desc::cie_xyz) into this translation unit's constant memory
void set_cie_xyz(const float *xyz, cudaStream_t s) {
    cudaMemcpyToSymbolAsync(PT_CIE_TABLE, xyz, sizeof(float) * 3 * B200PT_NSPEC, 0, cudaMemcpyHostToDevice, s);
}
// api.cu is compiled with the RGBSpectrum structs; RenderDev must not depend on the spectrum type
size_t render_dev_size() { return sizeof(RenderDev); }
#endif

}  // namespace B200PT_NS
