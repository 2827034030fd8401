// wbvh.h -- the acceleration structure that replaces the reference's binary
// LinearBVHNode array (accelerators/bvh.cpp:95-104): a 7-wide BVH with
// quantised child boxes in ONE 64-byte record per node (half a cache line, two
// 32-byte sectors, four 128-bit loads), after Ylitie, Karras, Laine, "Efficient
// Incoherent Ray Traversal on GPUs Through Compressed Wide BVHs" (HPG 2017).
//
// Why 7 children and 64 bytes: the traversal kernel streams every node from
// L2 (the working set of an incoherent wavefront is far beyond L1), so node
// bytes and their sector alignment bound the visit rate next to the ALU pipe.
// The 80-byte 8-wide record of round 1 straddled 3-4 sectors (112 bytes of L2
// traffic per visit on average); 7 children fit 64 aligned bytes.
//
// Node layout (little endian):
//   byte  0..11  float p[3]      origin of the node's grid = min corner of the node
//        12..14  uint8 e[3]      per-axis cell size = 2^(e-127)
//        15      uint8 imask     bit s set <=> slot s holds an inner child
//        16..19  uint32 child_base   index of the first inner child (inner children are contiguous, slot order)
//        20..21  uint16 lcount   2 bits per slot: triangles of a leaf child (0 = inner or empty slot)
//        22..35  uint8 zq[7][2]  per slot: (lo.z, hi.z) in cells
//        36..63  uint8 xyq[7][4] per slot: (lo.x, hi.x, lo.y, hi.y) in cells
// A child box is [p + lo*cell, p + hi*cell] per axis, a superset of the true
// box (rounded outward in exact arithmetic).  The (lo, hi) byte pair of one
// axis shares a 32-bit word, so the traversal kernel picks the near / far plane
// of a ray with one PRMT whose selector is a per-ray register -- no selects.
// An empty slot has lo = 255, hi = 0 on every axis, which no ray can hit.
// The first triangle of a node's leaf children lives in a side array
// (tri_base[node], read only when a leaf child was hit); the triangles of the
// leaf slots follow each other in slot order.
//
// Triangles are stored in leaf order as three float4: (p0, prim id) (p1,
// material id | flags) (p2, light id): everything shading needs sits in
// the 48 bytes traversal already touched.
#ifndef B200PT_WBVH_H
#define B200PT_WBVH_H

#include <cstdint>
#ifndef __CUDACC_RTC__
#include <vector>
#endif

#include "pt_platform.h"

namespace b200pt {

#define B200PT_WIDTH 7          // children per node
#define B200PT_EMPTY_LO 255u    // quantised box of an empty slot: lo > hi
#define B200PT_CELL_FLOOR 0x1p-17f  // smallest cell, relative to the largest |coordinate| of the tree (see wbvh_traverse.cuh)

struct alignas(64) WbvhNode {
    float p[3];
    uint8_t e[3];
    uint8_t imask;
    uint32_t child_base;
    uint16_t lcount;
    uint8_t zq[B200PT_WIDTH][2];
    uint8_t xyq[B200PT_WIDTH][4];
};
static_assert(sizeof(WbvhNode) == 64, "WbvhNode must be 64 bytes");

// flag bits of TriRecord::mat_flags above the 16-bit material id (DevSphere::mat_flags has the flip bit only)
#define B200PT_TRI_FLIP 0x10000u         // the geometric normal is flipped (reverseOrientation ^ transformSwapsHandedness)
#define B200PT_TRI_DEGENERATE 0x20000u   // Triangle::Intersect rejects it
#define B200PT_TRI_HAS_NORMALS 0x40000u  // per-vertex shading normals in DevScene::tri_n
#define B200PT_TRI_HAS_UVS 0x80000u      // uvs in DevScene::tri_uv
#define B200PT_TRI_INSTANCED 0x100000u   // object-space triangle of an instanced object
#define B200PT_TRI_ALPHA 0x200000u       // the mesh has an alpha or shadowalpha mask (b200pt_scene_set_alpha_masks)

struct alignas(16) TriRecord {  // 48 bytes
    float p0[3];
    uint32_t prim;
    float p1[3];
    uint32_t mat_flags;  // material id | B200PT_TRI_* flags
    float p2[3];
    int32_t light;
};
static_assert(sizeof(TriRecord) == 48, "TriRecord must be 48 bytes");

struct WbBox {
    float lo[3], hi[3];
};

B200_HD uint32_t wb_f2u(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
#endif
}
B200_HD float wb_u2f(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
B200_HD float wb_cell(uint8_t e) { return wb_u2f((uint32_t)e << 23); }

// Octant-ordered slot assignment (greedy on dot(centroid offset, octant direction)): visiting the slots by
// (slot XOR ray octant), highest first, then approximates front-to-back order.  childAt[s] = child or -1.
B200_HD void wbvh_assign_slots(const WbBox *box, int k, int *childAt) {
    WbBox nb = box[0];
    for (int i = 1; i < k; ++i)
        for (int a = 0; a < 3; ++a) {
            nb.lo[a] = box[i].lo[a] < nb.lo[a] ? box[i].lo[a] : nb.lo[a];
            nb.hi[a] = box[i].hi[a] > nb.hi[a] ? box[i].hi[a] : nb.hi[a];
        }
    float cost[B200PT_WIDTH][B200PT_WIDTH];
    for (int i = 0; i < k; ++i) {
        float cc[3];
        for (int a = 0; a < 3; ++a) cc[a] = 0.5f * box[i].lo[a] + 0.5f * box[i].hi[a] - (0.5f * nb.lo[a] + 0.5f * nb.hi[a]);
        for (int s = 0; s < B200PT_WIDTH; ++s)
            cost[i][s] = ((s & 1) ? cc[0] : -cc[0]) + ((s & 2) ? cc[1] : -cc[1]) + ((s & 4) ? cc[2] : -cc[2]);
    }
    bool slotUsed[B200PT_WIDTH], childDone[B200PT_WIDTH];
    for (int s = 0; s < B200PT_WIDTH; ++s) {
        childAt[s] = -1;
        slotUsed[s] = childDone[s] = false;
    }
    for (int round = 0; round < k; ++round) {
        int bi = -1, bs = -1;
        float bc = 0.f;
        for (int i = 0; i < k; ++i) {
            if (childDone[i]) continue;
            for (int s = 0; s < B200PT_WIDTH; ++s)
                if (!slotUsed[s] && (bi < 0 || cost[i][s] > bc)) {
                    bc = cost[i][s];
                    bi = i;
                    bs = s;
                }
        }
        childDone[bi] = true;
        slotUsed[bs] = true;
        childAt[bs] = bi;
    }
}

// Fills the geometric part of a node record: grid (p, e) over the union of the children, the quantised
// child boxes rounded outward, imask and lcount.  ntri[i] = 0 for an inner child, 1..3 for a leaf child.
// `cell_floor` (absolute) bounds the cell size from below so that the float error of the traversal's slab
// arithmetic stays a fraction of a cell: B200PT_CELL_FLOOR * largest |coordinate| of the tree.
B200_HD void wbvh_encode_node(const WbBox *box, const int *childAt, const uint8_t *ntri, float cell_floor, WbvhNode *out) {
    WbBox nb;
    bool any = false;
    for (int s = 0; s < B200PT_WIDTH; ++s) {
        const int i = childAt[s];
        if (i < 0) continue;
        for (int a = 0; a < 3; ++a) {
            nb.lo[a] = (!any || box[i].lo[a] < nb.lo[a]) ? box[i].lo[a] : nb.lo[a];
            nb.hi[a] = (!any || box[i].hi[a] > nb.hi[a]) ? box[i].hi[a] : nb.hi[a];
        }
        any = true;
    }
    if (!any)
        for (int a = 0; a < 3; ++a) nb.lo[a] = nb.hi[a] = 0.f;
    float cell[3];
    for (int a = 0; a < 3; ++a) {
        // smallest power of two with (hi - lo) / cell <= 254 (one spare cell for the rounding of this division)
        const float ext = nb.hi[a] - nb.lo[a];
        float need = ext / 254.f;
        if (!(need > cell_floor)) need = cell_floor;
        if (!(need > 1e-30f)) need = 1e-30f;
        uint32_t bits = wb_f2u(need);
        uint32_t be = (bits >> 23) & 0xffu;
        if (bits & 0x7fffffu) ++be;  // not an exact power of two: round up
        if (be < 1u) be = 1u;
        if (be > 254u) be = 254u;
        out->e[a] = (uint8_t)be;
        cell[a] = wb_cell((uint8_t)be);
        out->p[a] = nb.lo[a];
    }
    out->imask = 0;
    out->lcount = 0;
    for (int s = 0; s < B200PT_WIDTH; ++s) {
        const int i = childAt[s];
        uint8_t q[3][2];
        for (int a = 0; a < 3; ++a) {
            if (i < 0) {
                q[a][0] = (uint8_t)B200PT_EMPTY_LO;
                q[a][1] = 0;
                continue;
            }
            const double p = out->p[a], c = cell[a];
            float flo = (box[i].lo[a] - out->p[a]) / cell[a], fhi = (box[i].hi[a] - out->p[a]) / cell[a];
            int qlo = flo > 0.f ? (flo < 255.f ? (int)flo : 255) : 0;                 // floor for non-negative values
            int qhi = fhi > 0.f ? (fhi < 255.f ? (int)fhi + ((float)(int)fhi < fhi ? 1 : 0) : 255) : 0;  // ceil
            // outward in exact arithmetic (p + q * cell is exact in double)
            while (qlo > 0 && p + (double)qlo * c > (double)box[i].lo[a]) --qlo;
            while (qhi < 255 && p + (double)qhi * c < (double)box[i].hi[a]) ++qhi;
            q[a][0] = (uint8_t)qlo;
            q[a][1] = (uint8_t)qhi;
        }
        out->xyq[s][0] = q[0][0];
        out->xyq[s][1] = q[0][1];
        out->xyq[s][2] = q[1][0];
        out->xyq[s][3] = q[1][1];
        out->zq[s][0] = q[2][0];
        out->zq[s][1] = q[2][1];
        if (i >= 0) {
            if (ntri[i] == 0)
                out->imask |= (uint8_t)(1u << s);
            else
                out->lcount |= (uint16_t)((uint32_t)ntri[i] << (2 * s));
        }
    }
}

#ifndef __CUDACC_RTC__
struct Wbvh {
    std::vector<WbvhNode> nodes;     // node 0 is the root
    std::vector<uint32_t> tri_base;  // per node: first triangle of its leaf children
    std::vector<TriRecord> tris;     // leaf order; degenerate triangles (never hittable) at the end
    std::vector<uint32_t> prim_to_tri;  // original triangle index -> position in `tris`
    uint32_t n_in_leaves = 0;        // triangles referenced by leaves
    int max_depth = 0;               // depth of the wide tree (root = 1)
    float bounds_lo[3] = {0, 0, 0}, bounds_hi[3] = {0, 0, 0};  // bounds of the triangles in the tree
};

// Builds the wide BVH on the host: binned-SAH binary build (multi-threaded),
// SAH-optimal collapse to 7-wide, octant-ordered slot assignment, quantisation.
// `degenerate[i]` marks triangles the reference can never hit
// (shapes/triangle.cpp:304-312); they are kept out of the leaves.
void build_wbvh(const float *vertices, int64_t n_tris, const int32_t *material_id, const int32_t *light_id,
                const uint8_t *flip, const uint8_t *degenerate, int n_threads, Wbvh *out);

// Structural self-check used by the library after every build: every leaf
// triangle's exact bounds lie inside the decoded box of its slot and every
// inner child's content lies inside its parent's slot box.  Returns the
// number of violations.
int64_t validate_wbvh(const Wbvh &bvh);
#endif

}  // namespace b200pt
#endif
