// wbvh_traverse.cuh -- stack-based traversal of the 7-wide compressed BVH
// (wbvh.h), one ray per thread.  Replaces BVHAccel::Intersect / IntersectP
// (accelerators/bvh.cpp:662-738) + GeometricPrimitive::Intersect
// (core/primitive.cpp:116-130) + Triangle::Intersect / IntersectP
// (shapes/triangle.cpp:188-291, 427-517).
//
// What must match the reference bit for bit is the *result*: the hit triangle
// and (t, b0, b1, b2) come from the same watertight test with the same
// shrinking ray.tMax semantics (accept tScaled == tMax*det, primitive.cpp:120).
// The box tests only have to be conservative.
//
// Node test (round 2):
//   * the ray works in a box parameter s = (t - t0) / span, t0 = where it enters
//     the tree's bounds (0 if it starts inside), span = what is left of it
//     inside the bounds.  Every slab value is produced by one saturating FMA
//     (fma.rn.sat): the clamps max(t, 0) and min(t, tMax) of the slab test come
//     for free, and a child is hit iff max3(near) < min3(far) (strictly: boxes
//     entirely behind the origin or beyond the span clamp to 0 / 1 on both sides);
//   * a plane byte q is spliced into mantissa bits 8..15 of 2^15 by one PRMT:
//     the float 32768 + q, exactly; the -32768*a goes into the FMA's addend
//     (rounding error of that addend: a / 512, against half a cell for the
//     2^23 splice of round 1), so no slack cells are needed in the encoding;
//   * the near / far byte of each (lo, hi) pair is picked by the PRMT's
//     selector, a per-ray register: no selects, no octant-dependent branches;
//   * the hit bits of the inner children are permuted into traversal order
//     (slot XOR ray octant) by a 2 KB table (shared memory in k_trace).
// The float error of the slab values stays below 0.3 cells (the slack added to
// every box): cells are at least 2^-17 of the largest |coordinate| of the tree
// (wbvh.h) and a ray that starts outside the tree's bounds is first advanced to
// them, so |origin| stays of the order of the tree's extent -- also for rays
// transformed into the space of a small instanced object.
//
// Traversal state follows Ylitie et al. 2017: the stack holds "groups" --
// (child_base, hit bits | imask) for inner children still to visit -- and
// children are visited in the order (slot XOR ray octant), highest first, which
// the builder's slot assignment turns into an approximate front-to-back order.
#ifndef B200PT_WBVH_TRAVERSE_CUH
#define B200PT_WBVH_TRAVERSE_CUH

#include "pt_core.cuh"
#include "wbvh.h"

namespace B200PT_NS {

struct U4 {
    uint32_t x, y, z, w;
};
struct F4 {
    float x, y, z, w;
};
struct NodeWords {
    uint32_t w[16];
};

#ifdef __CUDA_ARCH__
B200_D U4 ld_u4(const U4 *p) {
    uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
    U4 r;
    r.x = v.x;
    r.y = v.y;
    r.z = v.z;
    r.w = v.w;
    return r;
}
B200_D F4 ld_f4(const F4 *p) {
    float4 v = __ldg(reinterpret_cast<const float4 *>(p));
    F4 r;
    r.x = v.x;
    r.y = v.y;
    r.z = v.z;
    r.w = v.w;
    return r;
}
// one 64-byte node = four 128-bit loads (LDG.E.128.CONSTANT; sm_90 has no 256-bit global load)
B200_D void ld_node(const U4 *nodes, uint32_t index, NodeWords *n) {
    const uint8_t *p = reinterpret_cast<const uint8_t *>(nodes) + (size_t)index * 64;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p + 16 * j));
        n->w[4 * j] = v.x;
        n->w[4 * j + 1] = v.y;
        n->w[4 * j + 2] = v.z;
        n->w[4 * j + 3] = v.w;
    }
}
B200_D float fma_any(float a, float b, float c) { return __fmaf_rn(a, b, c); }
B200_D float fma_sat(float a, float b, float c) {
    float r;
    asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
    return r;
}
// 32768 + (the byte of w that `sel` names), see trav_init for the selectors
B200_D float plane_2p15(uint32_t w, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(w), "n"(0x47000000), "r"(sel));
    return __uint_as_float(r);
}
B200_D float box_max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
B200_D float box_min3(float a, float b, float c) { return fminf(fminf(a, b), c); }
// the word with the bytes of each 16-bit half swapped: (lo, hi) pairs become (hi, lo)
B200_D uint32_t swap_pairs(uint32_t w) { return __byte_perm(w, 0u, 0x2301u); }
// m |= bit if a < b, as one compare and one predicated OR
template <uint32_t BIT>
B200_D void or_if_less(uint32_t &m, float a, float b) {
    asm("{\n\t.reg .pred p;\n\tsetp.lt.f32 p, %1, %2;\n\t@p or.b32 %0, %0, %3;\n\t}" : "+r"(m) : "f"(a), "f"(b), "n"(BIT));
}
// B200PT_BOX_SLACK with the sign of x
B200_D float slack_signed(float x) { return __uint_as_float(0x3e99999au | (__float_as_uint(x) & 0x80000000u)); }
B200_D int msb32(uint32_t v) { return 31 - __clz((int)v); }
B200_D int popc32(uint32_t v) { return __popc(v); }
#else
inline U4 ld_u4(const U4 *p) { return *p; }
inline F4 ld_f4(const F4 *p) { return *p; }
inline void ld_node(const U4 *nodes, uint32_t index, NodeWords *n) { memcpy(n->w, nodes + (size_t)index * 4, 64); }
inline float fma_any(float a, float b, float c) { return fmaf(a, b, c); }
inline float fma_sat(float a, float b, float c) {
    const float r = fmaf(a, b, c);
    return r > 0.f ? (r < 1.f ? r : 1.f) : 0.f;  // NaN -> 0 like the instruction
}
inline float plane_2p15(uint32_t w, uint32_t sel) {
    return uint_as_float(0x47000000u | (((w >> (8 * ((sel >> 4) & 3u))) & 0xffu) << 8));
}
inline float box_max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
inline float box_min3(float a, float b, float c) { return fminf(fminf(a, b), c); }
template <uint32_t BIT>
inline void or_if_less(uint32_t &m, float a, float b) {
    if (a < b) m |= BIT;
}
inline uint32_t swap_pairs(uint32_t w) { return ((w & 0x00ff00ffu) << 8) | ((w >> 8) & 0x00ff00ffu); }
inline float slack_signed(float x) { return uint_as_float(0x3e99999au | (float_as_uint(x) & 0x80000000u)); }
inline int msb32(uint32_t v) { return 31 - __builtin_clz(v); }
inline int popc32(uint32_t v) { return __builtin_popcount(v); }
#endif

#define B200PT_STACK 48
#define B200PT_MISS 0xffffffffu
#define B200PT_BOX_SLACK 0.3f  // cells, see the header (0x3e99999a, slack_signed)

struct TraceCounters {
    uint32_t nodes, tris;
};

// bounds of the tree a ray is traversed against (slightly padded) and the length scale that floors a ray's span
struct TravBounds {
    float lo[3], hi[3], scale;
};

B200_HD float safe_rcp_dir(float d) {
    // keeps the sign of d, avoids inf/NaN in the slab arithmetic for axis-parallel rays
    float a = pt_abs(d);
    if (!(a > 1e-20f)) d = (float_as_uint(d) & 0x80000000u) ? -1e-20f : 1e-20f;
    return 1.0f / d;
}

// permutation of the 7 slot bits into traversal order: bit s -> bit (s ^ octinv)
B200_HD uint32_t permute_slots(uint32_t m, uint32_t octinv) {
    uint32_t r = 0;
    for (uint32_t s = 0; s < 8; ++s)
        if (m & (1u << s)) r |= 1u << (s ^ octinv);
    return r;
}
#define B200PT_LUT_BYTES 2048  // table of permute_slots: lut[octinv << 8 | m]

// Per-ray traversal state, in two parts.  `Trav` is what the node test reads at every step (it lives in
// registers); `TravRay` is the ray as the triangle test sees it plus the result so far -- k_trace keeps it in
// shared memory and fetches it for the (much rarer) triangle phase.
// One step = "take the next child group: fetch its node and test the seven children, then intersect the
// leaf triangles that were hit".
struct Trav {
    // ---- box test
    float idx, idy, idz;   // 1 / d, per unit of the box parameter
    float oix, oiy, oiz;   // (o + t0 d) * (idx, idy, idz)
    uint32_t sel[4];       // PRMT selectors of the NEAR byte: x, y (bytes 0-1 / 2-3 of a slot's xy word), z pair at bytes 0-1, at
                           // bytes 2-3; the far byte is fetched with the same selector from the word with its byte pairs swapped
    uint32_t octinv;       // 7 - ray octant
    // ---- position in the tree
    uint32_t cur_x, cur_y;
    int sp;                // stack pointer; bit 30 is set when a push was dropped because the stack was full (reported,
                           // never silent: B200PT_SP_OVERFLOW)
};
#define B200PT_SP_OVERFLOW 0x40000000
#define B200PT_SP_MASK 0x3fffffff
struct TravRay {
    V3 o;
    RayShear sh;
    float tmax;
    uint32_t best;
    TriHit hit;
    float t0;              // box parameter = (t - t0) / span
    // what trav_rescale needs when a closest hit shortens the ray: the unscaled reciprocal direction, the advanced
    // origin times it, and the floor of the span
    float iu[3], ou[3], span_floor;
};
// The stack of postponed child groups lives in its own object so that the scalar
// state above stays in registers (a struct with a dynamically indexed array is
// placed in local memory as a whole).
struct TravStack {
    uint32_t x[B200PT_STACK], y[B200PT_STACK];
    B200_HD void push(int sp, uint32_t gx, uint32_t gy) {
        x[sp] = gx;
        y[sp] = gy;
    }
    B200_HD void pop(int sp, uint32_t *gx, uint32_t *gy) const {
        *gx = x[sp];
        *gy = y[sp];
    }
};

// The box parameter ends (s = 1) a little beyond `tEnd`, the ray's current tMax (or where it leaves the bounds): the span
// is a little longer than tEnd - t0 and never shorter than 2^-30 of the tree's extent (keeps every product finite).
// Called once per ray and again whenever a closest hit shortens the ray -- from the unscaled values, so nothing drifts.
B200_HD void trav_rescale(Trav &T, const TravRay &R, float tEnd) {
    float span = (tEnd - R.t0) * 1.001f + 0x1p-20f * tEnd;
    if (!(span > R.span_floor)) span = R.span_floor;
    if (!(span > 1e-30f)) span = 1e-30f;
    const float inv = 1.0f / span;
    T.idx = R.iu[0] * inv;
    T.idy = R.iu[1] * inv;
    T.idz = R.iu[2] * inv;
    T.oix = R.ou[0] * inv;
    T.oiy = R.ou[1] * inv;
    T.oiz = R.ou[2] * inv;
}

B200_HD void trav_init(Trav &T, TravRay &R, const V3 &o, const V3 &d, float rayTMax, const TravBounds &B) {
    R.o = o;
    R.sh = make_shear(d);
    R.tmax = rayTMax;
    R.best = B200PT_MISS;
    R.hit.t = R.hit.b0 = R.hit.b1 = R.hit.b2 = 0.f;
    T.sp = 0;
    T.cur_x = 0u;
    T.cur_y = 0u;  // nothing to do unless the ray meets the bounds
    const float ix = safe_rcp_dir(d.x), iy = safe_rcp_dir(d.y), iz = safe_rcp_dir(d.z);
    // the octant follows the sign BIT, like safe_rcp_dir does: a component of -0.0 (mirrored instances, reflections)
    // must pick the same near / far planes as the sign of its reciprocal
    const uint32_t nx = float_as_uint(d.x) >> 31, ny = float_as_uint(d.y) >> 31, nz = float_as_uint(d.z) >> 31;
    const uint32_t oct = nx | (ny << 1) | (nz << 2);
    T.octinv = 7u - oct;
    // PRMT selector 0x74B4: result bytes (3..0) = (0x47, 0x00, byte B of the node word, 0x00) = the float 32768 + byte
    T.sel[0] = 0x7404u | (nx << 4);
    T.sel[1] = 0x7424u | (ny << 4);
    T.sel[2] = 0x7404u | (nz << 4);
    T.sel[3] = 0x7424u | (nz << 4);
    // the part of the ray inside the bounds: [t0, t1] (the clip itself widened by its own rounding)
    const float ax0 = (B.lo[0] - o.x) * ix, ax1 = (B.hi[0] - o.x) * ix;
    const float ay0 = (B.lo[1] - o.y) * iy, ay1 = (B.hi[1] - o.y) * iy;
    const float az0 = (B.lo[2] - o.z) * iz, az1 = (B.hi[2] - o.z) * iz;
    const float tEnter = box_max3(pt_min(ax0, ax1), pt_min(ay0, ay1), pt_min(az0, az1)) * (1.f - 0x1p-18f);
    const float tExit = box_min3(pt_max(ax0, ax1), pt_max(ay0, ay1), pt_max(az0, az1)) * (1.f + 0x1p-18f);
    const float t0 = tEnter > 0.f ? tEnter : 0.f;
    const float t1 = tExit < rayTMax ? tExit : rayTMax;
    R.t0 = t0;
    R.iu[0] = ix;
    R.iu[1] = iy;
    R.iu[2] = iz;
    R.ou[0] = R.ou[1] = R.ou[2] = 0.f;
    R.span_floor = 0x1p-30f * B.scale;
    T.idx = T.idy = T.idz = T.oix = T.oiy = T.oiz = 0.f;
    if (!(t0 <= t1)) return;  // misses the bounds (or NaN): no traversal at all
    const float obx = t0 > 0.f ? fma_any(d.x, t0, o.x) : o.x, oby = t0 > 0.f ? fma_any(d.y, t0, o.y) : o.y,
                obz = t0 > 0.f ? fma_any(d.z, t0, o.z) : o.z;
    R.ou[0] = obx * ix;
    R.ou[1] = oby * iy;
    R.ou[2] = obz * iz;
    trav_rescale(T, R, t1);
    T.cur_y = 0x80000000u;  // the root as a one-child group
}

#define B200PT_SLOT(S, WXY, WXYS, WZ, WZS, ZSEL)                                                                     \
    {                                                                                                                \
        const float tn = box_max3(fma_sat(plane_2p15(WXY, T.sel[0]), ax, cnx), fma_sat(plane_2p15(WXY, T.sel[1]), ay, cny), \
                                  fma_sat(plane_2p15(WZ, T.sel[ZSEL]), az, cnz));                                    \
        const float tf = box_min3(fma_sat(plane_2p15(WXYS, T.sel[0]), ax, cfx), fma_sat(plane_2p15(WXYS, T.sel[1]), ay, cfy), \
                                  fma_sat(plane_2p15(WZS, T.sel[ZSEL]), az, cfz));                                   \
        or_if_less<(1u << S)>(m, tn, tf);                                                                            \
    }

// Node phase: take the next inner child of the current group, fetch its node, test the seven
// children.  Leaves the hit inner children in T.cur and returns the hit leaf children as a
// leaf group (*tg_x = the node, *tg_y = hit leaf slots | lcount << 8, 0 if none).  Requires T.cur to be a node group.
// (CLOSEST is kept for the callers' sake: a closest hit rescales the box parameter, trav_rescale, so the test itself is
// the same for both kinds of ray.)
template <bool CLOSEST, bool COUNT>
B200_HD void trav_node_phase(Trav &T, TravStack &S, const U4 *__restrict__ nodes, const uint32_t *__restrict__ /*tri_base*/,
                             const uint8_t *lut, uint32_t *tg_x, uint32_t *tg_y, TraceCounters *ctr) {
    const uint32_t hits = T.cur_y;
    const int bit = msb32(hits);
    T.cur_y &= ~(1u << bit);
    if (T.cur_y & 0xff000000u) {
        if ((T.sp & B200PT_SP_MASK) < B200PT_STACK) {
            S.push(T.sp & B200PT_SP_MASK, T.cur_x, T.cur_y);
            ++T.sp;
        } else {
            T.sp |= B200PT_SP_OVERFLOW;
        }
    }
    const uint32_t slot = ((uint32_t)(bit - 24)) ^ T.octinv;
    const uint32_t rel = (uint32_t)popc32(hits & 0xffu & ((1u << slot) - 1u));
    const uint32_t ni = T.cur_x + rel;
    NodeWords n;
    ld_node(nodes, ni, &n);
    if (COUNT) ctr->nodes++;
    // w0-2: p   w3: e.x e.y e.z imask   w4: child_base   w5: lcount | z pair of slot 0   w6-8: z pairs of slots 1..6
    // w9+s: (lo.x hi.x lo.y hi.y) of slot s.  plane(q) = p + q*cell, in box-parameter units q*a + k with a = cell/d,
    // k = (p - o)/d; the byte arrives as 32768 + q, the slack of B200PT_BOX_SLACK cells moves the near planes towards
    // the ray and the far planes away from it.
    const float ax = uint_as_float((n.w[3] & 0xffu) << 23) * T.idx;
    const float ay = uint_as_float(((n.w[3] >> 8) & 0xffu) << 23) * T.idy;
    const float az = uint_as_float(((n.w[3] >> 16) & 0xffu) << 23) * T.idz;
    const float c0x = fma_any(-32768.0f, ax, fma_any(uint_as_float(n.w[0]), T.idx, -T.oix));
    const float c0y = fma_any(-32768.0f, ay, fma_any(uint_as_float(n.w[1]), T.idy, -T.oiy));
    const float c0z = fma_any(-32768.0f, az, fma_any(uint_as_float(n.w[2]), T.idz, -T.oiz));
    // slack: 0.3 |a| towards the ray for the near planes, away from it for the far ones (a has the sign of the direction)
    const float sx = slack_signed(T.idx), sy = slack_signed(T.idy), sz = slack_signed(T.idz);
    const float cnx = fma_any(-sx, ax, c0x), cny = fma_any(-sy, ay, c0y), cnz = fma_any(-sz, az, c0z);
    const float cfx = fma_any(sx, ax, c0x), cfy = fma_any(sy, ay, c0y), cfz = fma_any(sz, az, c0z);
    const uint32_t z0 = swap_pairs(n.w[5]), z1 = swap_pairs(n.w[6]), z2 = swap_pairs(n.w[7]), z3 = swap_pairs(n.w[8]);
    uint32_t m = 0;
    B200PT_SLOT(0, n.w[9], swap_pairs(n.w[9]), n.w[5], z0, 3)
    B200PT_SLOT(1, n.w[10], swap_pairs(n.w[10]), n.w[6], z1, 2)
    B200PT_SLOT(2, n.w[11], swap_pairs(n.w[11]), n.w[6], z1, 3)
    B200PT_SLOT(3, n.w[12], swap_pairs(n.w[12]), n.w[7], z2, 2)
    B200PT_SLOT(4, n.w[13], swap_pairs(n.w[13]), n.w[7], z2, 3)
    B200PT_SLOT(5, n.w[14], swap_pairs(n.w[14]), n.w[8], z3, 2)
    B200PT_SLOT(6, n.w[15], swap_pairs(n.w[15]), n.w[8], z3, 3)
    const uint32_t imask = n.w[3] >> 24;
    const uint32_t mi = m & imask;
#ifdef __CUDA_ARCH__
    const uint32_t pm = lut[(T.octinv << 8) | mi];
#else
    (void)lut;
    const uint32_t pm = permute_slots(mi, T.octinv);
#endif
    T.cur_x = n.w[4];
    T.cur_y = (pm << 24) | imask;
    // leaf children that were hit: the node's number and (slot bits | lcount << 8); trav_tri_phase turns them into triangles
    const uint32_t ml = m & ~imask;
    *tg_x = ni;
    *tg_y = ml ? (ml | ((n.w[5] & 0xffffu) << 8)) : 0u;
}
#undef B200PT_SLOT

// Triangle phase: exact watertight tests of a triangle group.  Returns true if ANY_HIT found a hit.
// A leaf group of the node phase (node, hit leaf slots | lcount << 8) as a triangle group: *tg_x = first triangle of the
// node's leaf children, *tg_y = bit per triangle (the triangles of the leaf slots follow each other in slot order).
B200_HD void leaf_group_triangles(const uint32_t *__restrict__ tri_base, uint32_t lg_x, uint32_t lg_y, uint32_t *tg_x, uint32_t *tg_y) {
    *tg_x = 0;
    *tg_y = 0;
    if (!lg_y) return;
    *tg_x = tri_base[lg_x];
    const uint32_t lc = lg_y >> 8;
    uint32_t ml = lg_y & 0x7fu, bits = 0;
    do {
        const int s = msb32(ml);
        ml &= ~(1u << s);
        const uint32_t below = lc & ((1u << (2 * s)) - 1u);
        const uint32_t off = (uint32_t)popc32(below & 0x5555u) + 2u * (uint32_t)popc32(below & 0xaaaau);
        bits |= ((1u << ((lc >> (2 * s)) & 3u)) - 1u) << off;
    } while (ml);
    *tg_y = bits;
}

// Triangles without alpha masks: the watertight test alone decides.  Every scene without masks runs this.
struct NoAlpha {
    static constexpr bool enabled = false;
    template <class ARGS>
    B200_HD static NoAlpha of(const ARGS &) {  // (a launch's arguments, as AlphaTest::of takes them)
        return NoAlpha();
    }
    B200_HD NoAlpha at(uint32_t) const { return *this; }
    B200_HD bool rejects(bool, uint32_t, uint32_t, uint32_t, const TriHit &) const { return false; }
};

// ALPHA (see AlphaTest in kernels.cu) rejects a candidate the test accepted when its mesh's mask evaluates to exactly 0
// (Triangle::Intersect / IntersectP, shapes/triangle.cpp:332-337, 531-570).  A rejected candidate does not shorten the ray.
// Only triangles flagged B200PT_TRI_ALPHA are looked up, from the flag word the test loads anyway.
template <bool ANY_HIT, bool COUNT, class ALPHA = NoAlpha>
B200_HD bool trav_tri_phase(TravRay &R, const uint32_t *__restrict__ tri_base, const F4 *__restrict__ tris, uint32_t lg_x,
                            uint32_t lg_y, TraceCounters *ctr, const ALPHA &alpha = ALPHA()) {
    uint32_t tg_x, tg_y;
    leaf_group_triangles(tri_base, lg_x, lg_y, &tg_x, &tg_y);
    while (tg_y) {
        const int j = msb32(tg_y);
        tg_y &= ~(1u << j);
        const uint32_t ti = tg_x + (uint32_t)j;
        const F4 *tp = tris + (size_t)ti * 3;
        const F4 v0 = ld_f4(tp), v1 = ld_f4(tp + 1), v2 = ld_f4(tp + 2);
        if (COUNT) ctr->tris++;
        TriHit h;
        if (triangle_test(mk(v0.x, v0.y, v0.z), mk(v1.x, v1.y, v1.z), mk(v2.x, v2.y, v2.z), R.o, R.sh, R.tmax, &h)) {
            if (ALPHA::enabled && (float_as_uint(v1.w) & B200PT_TRI_ALPHA) &&
                alpha.rejects(ANY_HIT, ti, float_as_uint(v0.w), float_as_uint(v1.w), h))
                continue;
            R.tmax = h.t;  // primitive.cpp:120 (the caller rescales the box parameter: trav_rescale)
            R.best = ti;
            R.hit = h;
            if (ANY_HIT) return true;
        }
    }
    return false;
}

// Pops the next node group if the current one is exhausted; false when nothing is left.
B200_HD bool trav_next_group(Trav &T, TravStack &S) {
    if ((T.cur_y & 0xff000000u) == 0) {
        if ((T.sp & B200PT_SP_MASK) == 0) return false;
        --T.sp;
        S.pop(T.sp & B200PT_SP_MASK, &T.cur_x, &T.cur_y);
    }
    return true;
}

// One complete step (node phase, then its triangles at once).  Returns true when the traversal
// is complete (closest hit known / any hit found / nothing left).
template <bool ANY_HIT, bool COUNT, class ALPHA = NoAlpha>
B200_HD bool trav_step(Trav &T, TravRay &R, TravStack &S, const U4 *__restrict__ nodes, const uint32_t *__restrict__ tri_base,
                        const F4 *__restrict__ tris, const uint8_t *lut, TraceCounters *ctr, const ALPHA &alpha = ALPHA()) {
    uint32_t tg_x = 0, tg_y = 0;
    if (T.cur_y & 0xff000000u) trav_node_phase<!ANY_HIT, COUNT>(T, S, nodes, tri_base, lut, &tg_x, &tg_y, ctr);
    const float before = R.tmax;
    if (trav_tri_phase<ANY_HIT, COUNT>(R, tri_base, tris, tg_x, tg_y, ctr, alpha)) return true;
    if (R.tmax != before) trav_rescale(T, R, R.tmax);
    return !trav_next_group(T, S);
}

// Whole traversal of one ray (used by the CPU pre-flight and the simple entry points).
// Returns the leaf-order index of the closest (ANY_HIT: of some) hit triangle or
// B200PT_MISS; *hit receives (t, b0, b1, b2) of the accepted intersection.
template <bool ANY_HIT, bool COUNT, class ALPHA = NoAlpha>
B200_HD uint32_t traverse_wbvh(const U4 *__restrict__ nodes, const uint32_t *__restrict__ tri_base, const F4 *__restrict__ tris,
                               const TravBounds &B, const uint8_t *lut, const V3 &o, const V3 &d, float rayTMax, TriHit *hit,
                               TraceCounters *ctr, uint32_t *overflow = nullptr, const ALPHA &alpha = ALPHA()) {
    Trav T;
    TravRay R;
    TravStack S;
    trav_init(T, R, o, d, rayTMax, B);
    if (T.cur_y & 0xff000000u)
        while (!trav_step<ANY_HIT, COUNT>(T, R, S, nodes, tri_base, tris, lut, ctr, alpha)) {
        }
    *hit = R.hit;
    if (overflow && (T.sp & B200PT_SP_OVERFLOW)) *overflow += 1;
    return R.best;
}

}  // namespace B200PT_NS
#endif
