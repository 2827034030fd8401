// lbvh.cuh -- the per-element steps of the on-device builder of the 7-wide BVH (wbvh.h)
// (SURVEY 8f row 1: replaces the host SAH build of wbvh_build.cpp, and with it
// BVHAccel's constructor accelerators/bvh.cpp:183-225, when build time matters
// more than tree quality).  The reference's own parallel design is HLBVH
// (bvh.cpp:404-638: Morton codes -> radix sort -> treelets -> SAH over
// treelets); here the whole tree comes from the Morton order:
//
//   1. lbvh_prep        triangle bounds / centroid, degenerate + non-finite filter
//   2. lbvh_key         63-bit Morton code of the centroid (21 bits per axis)
//      radix sort of (key, triangle) pairs
//   3. lbvh_karras      binary radix tree over the sorted keys (Karras 2012:
//                       one thread per internal node, no synchronisation)
//   4. lbvh_fit_*       bottom-up bounds (second arrival at a node continues)
//   5. lbvh_collapse    top-down, one thread per wide node: open the child with
//                       the largest surface area until 7 slots are used,
//                       subtrees of <= 3 triangles become leaf children;
//                       octant-ordered slots + quantisation exactly like the
//                       host builder; triangle records written in leaf order
//
// Every step is a B200_HD function of an element index so that
// tests/host_preflight.cpp can run the identical code on the CPU (sequentially)
// and check the result with validate_wbvh and against the oracle before GPU
// time is spent.  The tree's topology is not part of the parity contract:
// closest hits are decided by the exact triangle test.
#ifndef B200PT_LBVH_CUH
#define B200PT_LBVH_CUH

#include "wbvh.h"
#include "pt_core.cuh"

namespace b200pt {

#ifndef LBVH_OPEN_SMALL
#define LBVH_OPEN_SMALL 2  // also open subtrees of 2-3 triangles while the node has free slots (fewer triangle tests)
#endif

struct LbvhItem {
    int32_t node2;   // binary node to expand (internal id, or ~leaf for a single-triangle root)
    uint32_t wide;   // index of the wide node to fill
};

struct LbvhCtx {
    // ---- input (scene descriptor arrays)
    const float *vertices;        // [n][3][3]
    const int32_t *material_id, *light_id;
    const uint8_t *flip, *vertex_flags;
    const float *uvs;             // optional [n][3][2] (degenerate test + flag)
    int has_normals, has_uvs;
    int64_t n;
    // ---- pass 1/2
    uint32_t *valid_idx;          // triangles that enter the tree
    uint32_t *n_valid;            // counter
    int32_t *cbounds;             // centroid bounds as ordered ints: min xyz, max xyz; then the triangles' bounds [6..11]
    float cell_floor;             // smallest cell of the quantisation grids (set by the host before the collapse)
    uint64_t *keys;               // Morton keys (sorted in place with `sorted`)
    uint32_t *sorted;             // triangle ids in key order
    int64_t m;                    // = *n_valid, set by the host before pass 3
    // ---- binary radix tree: internal nodes 0..m-2, leaf j = sorted position j
    int32_t *left, *right;        // >= 0 internal, < 0: ~leaf
    int32_t *parent;              // [2m-1]: internal i at i, leaf j at (m-1)+j; root's parent = -1
    int32_t *first, *last;        // key range of internal node
    float *nbox;                  // [m-1][6]
    uint32_t *arrivals;           // [m-1]
    // ---- output
    WbvhNode *nodes;
    uint32_t *tri_base;           // parallel to nodes
    uint64_t node_cap;            // allocated wide nodes (writes beyond it are dropped; the driver reports the overflow)
    TriRecord *tris;
    uint32_t *prim_to_tri;        // [n], 0xffffffff until placed
    uint32_t *n_nodes, *n_tris;   // allocation counters
    // ---- frontier of the collapse
    const LbvhItem *q_in;
    LbvhItem *q_out;
    uint32_t *q_out_count;
};

B200_HD uint32_t lb_atomic_add(uint32_t *p, uint32_t v) {
#ifdef __CUDA_ARCH__
    return atomicAdd(p, v);
#else
    const uint32_t old = *p;
    *p += v;
    return old;
#endif
}
// order-preserving float <-> int map so that integer atomicMin/Max order floats
B200_HD int32_t lb_float_to_ordered(float f) {
    const int32_t i = (int32_t)float_as_uint(f);
    return i >= 0 ? i : (int32_t)(i ^ 0x7fffffff);
}
B200_HD float lb_ordered_to_float(int32_t i) { return uint_as_float((uint32_t)(i >= 0 ? i : (i ^ 0x7fffffff))); }
B200_HD void lb_atomic_min(int32_t *p, int32_t v) {
#ifdef __CUDA_ARCH__
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
B200_HD void lb_atomic_max(int32_t *p, int32_t v) {
#ifdef __CUDA_ARCH__
    atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}
B200_HD int lb_clz64(uint64_t v) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)v);
#else
    return v ? __builtin_clzll(v) : 64;
#endif
}
B200_HD int lb_clz32(uint32_t v) {
#ifdef __CUDA_ARCH__
    return __clz((int)v);
#else
    return v ? __builtin_clz(v) : 32;
#endif
}

struct LbBox {
    float lo[3], hi[3];
};
B200_HD void lb_tri_box(const float *v, LbBox *b) {
    for (int a = 0; a < 3; ++a) {
        b->lo[a] = pt_min(v[a], pt_min(v[3 + a], v[6 + a]));
        b->hi[a] = pt_max(v[a], pt_max(v[3 + a], v[6 + a]));
    }
}
B200_HD float lb_half_area(const LbBox &b) {
    const float dx = b.hi[0] - b.lo[0], dy = b.hi[1] - b.lo[1], dz = b.hi[2] - b.lo[2];
    if (!(dx >= 0) || !(dy >= 0) || !(dz >= 0)) return 0.f;
    return dx * dy + dy * dz + dz * dx;
}
B200_HD bool lb_finite(float f) { return (float_as_uint(f) & 0x7f800000u) != 0x7f800000u; }

// ---- 1. per triangle: does it enter the tree?  (shapes/triangle.cpp:304-312 for the degenerate rule)
B200_HD void lbvh_prep(const LbvhCtx &c, int64_t i) {
    const float *v = c.vertices + 9 * i;
    c.prim_to_tri[i] = 0xffffffffu;
    LbBox b;
    lb_tri_box(v, &b);
    bool ok = true;
    for (int a = 0; a < 3; ++a) ok = ok && lb_finite(b.lo[a]) && lb_finite(b.hi[a]);
    TriShading sh;
    default_shading(&sh);
    const uint8_t vf = c.vertex_flags ? c.vertex_flags[i] : 3;
    if (c.uvs && (vf & 2))
        for (int k = 0; k < 6; ++k) sh.uv[k] = c.uvs[6 * i + k];
    V3 dpdu, dpdv;
    const bool degenerate =
        !triangle_partials(mk(v[0], v[1], v[2]), mk(v[3], v[4], v[5]), mk(v[6], v[7], v[8]), sh.uv, &dpdu, &dpdv);
    if (!ok || degenerate) return;
    const uint32_t pos = lb_atomic_add(c.n_valid, 1u);
    c.valid_idx[pos] = (uint32_t)i;
    for (int a = 0; a < 3; ++a) {
        const float cen = 0.5f * b.lo[a] + 0.5f * b.hi[a];
        lb_atomic_min(c.cbounds + a, lb_float_to_ordered(cen));
        lb_atomic_max(c.cbounds + 3 + a, lb_float_to_ordered(cen));
        lb_atomic_min(c.cbounds + 6 + a, lb_float_to_ordered(b.lo[a]));
        lb_atomic_max(c.cbounds + 9 + a, lb_float_to_ordered(b.hi[a]));
    }
}

B200_HD uint64_t lb_expand21(uint32_t v) {  // spread the low 21 bits: one bit every third position
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}
// ---- 2. Morton key of valid triangle k
B200_HD void lbvh_key(const LbvhCtx &c, int64_t k) {
    const uint32_t i = c.valid_idx[k];
    LbBox b;
    lb_tri_box(c.vertices + 9 * (int64_t)i, &b);
    uint64_t key = 0;
    for (int a = 0; a < 3; ++a) {
        const float lo = lb_ordered_to_float(c.cbounds[a]), hi = lb_ordered_to_float(c.cbounds[3 + a]);
        const float cen = 0.5f * b.lo[a] + 0.5f * b.hi[a];
        float t = hi > lo ? (cen - lo) / (hi - lo) : 0.f;
        t = pt_min(pt_max(t, 0.f), 1.f);
        const uint32_t q = (uint32_t)pt_min(t * 2097152.f, 2097151.f);
        key |= lb_expand21(q) << (2 - a);  // x is the most significant bit of every triple
    }
    c.keys[k] = key;
    c.sorted[k] = i;
}

// ---- 3. binary radix tree (Karras 2012, "Maximizing Parallelism in the Construction of BVHs, Octrees, and k-d Trees")
B200_HD int lb_delta(const LbvhCtx &c, int64_t i, int64_t j) {
    if (j < 0 || j >= c.m) return -1;
    const uint64_t a = c.keys[i], b = c.keys[j];
    if (a == b) return 64 + lb_clz32((uint32_t)i ^ (uint32_t)j);
    return lb_clz64(a ^ b);
}
B200_HD void lbvh_karras(const LbvhCtx &c, int64_t i) {
    const int d = (lb_delta(c, i, i + 1) - lb_delta(c, i, i - 1)) >= 0 ? 1 : -1;
    const int dmin = lb_delta(c, i, i - d);
    int64_t lmax = 2;
    while (lb_delta(c, i, i + lmax * d) > dmin) lmax *= 2;
    int64_t l = 0;
    for (int64_t t = lmax / 2; t >= 1; t /= 2)
        if (lb_delta(c, i, i + (l + t) * d) > dmin) l += t;
    const int64_t j = i + l * d;
    const int dnode = lb_delta(c, i, j);
    int64_t s = 0, t = l;
    do {
        t = (t + 1) / 2;
        if (lb_delta(c, i, i + (s + t) * d) > dnode) s += t;
    } while (t > 1);
    const int64_t gamma = i + s * d + (d < 0 ? -1 : 0);
    const int64_t lo = i < j ? i : j, hi = i < j ? j : i;
    const int32_t L = (lo == gamma) ? ~(int32_t)gamma : (int32_t)gamma;
    const int32_t R = (hi == gamma + 1) ? ~(int32_t)(gamma + 1) : (int32_t)(gamma + 1);
    c.left[i] = L;
    c.right[i] = R;
    c.first[i] = (int32_t)lo;
    c.last[i] = (int32_t)hi;
    c.parent[L >= 0 ? L : (c.m - 1) + (int64_t)(~L)] = (int32_t)i;
    c.parent[R >= 0 ? R : (c.m - 1) + (int64_t)(~R)] = (int32_t)i;
    if (i == 0) c.parent[0] = -1;
    c.arrivals[i] = 0u;
}

// bounds of a binary child: a leaf's triangle or an internal node's fitted box
B200_HD void lb_child_box(const LbvhCtx &c, int32_t child, LbBox *b) {
    if (child < 0) {
        lb_tri_box(c.vertices + 9 * (int64_t)c.sorted[~child], b);
    } else {
        const float *p = c.nbox + 6 * (int64_t)child;
        for (int a = 0; a < 3; ++a) {
            b->lo[a] = p[a];
            b->hi[a] = p[3 + a];
        }
    }
}
B200_HD void lb_fit_node(const LbvhCtx &c, int32_t node) {
    LbBox a, b;
    lb_child_box(c, c.left[node], &a);
    lb_child_box(c, c.right[node], &b);
    float *p = c.nbox + 6 * (int64_t)node;
    for (int k = 0; k < 3; ++k) {
        p[k] = pt_min(a.lo[k], b.lo[k]);
        p[3 + k] = pt_max(a.hi[k], b.hi[k]);
    }
}
#ifdef __CUDACC__
// ---- 4. (device) bottom-up from leaf j: the second thread to arrive at a node fits it and continues
__device__ __forceinline__ void lbvh_fit_from_leaf(const LbvhCtx &c, int64_t j) {
    int32_t node = c.parent[(c.m - 1) + j];
    while (node >= 0) {
        __threadfence();
        if (atomicAdd(c.arrivals + node, 1u) == 0u) return;
        lb_fit_node(c, node);
        node = c.parent[node];
    }
}
#endif

B200_HD int32_t lb_count(const LbvhCtx &c, int32_t child) { return child < 0 ? 1 : c.last[child] - c.first[child] + 1; }

// ---- 5. one wide node: choose its children, place them, quantise, write triangles, queue inner children
B200_HD void lbvh_collapse(const LbvhCtx &c, const LbvhItem &it) {
    constexpr int W = B200PT_WIDTH;
    int32_t ch[W];
    LbBox box[W];
    int k = 0;
    if (it.node2 < 0) {
        ch[k] = it.node2;  // a single triangle: one leaf child of the root
        lb_child_box(c, it.node2, &box[k]);
        ++k;
    } else {
        ch[0] = c.left[it.node2];
        ch[1] = c.right[it.node2];
        lb_child_box(c, ch[0], &box[0]);
        lb_child_box(c, ch[1], &box[1]);
        k = 2;
        while (k < W) {
            int best = -1;
            float bestArea = -1.f;
            for (int i = 0; i < k; ++i) {
                if (ch[i] < 0 || (LBVH_OPEN_SMALL == 0 && lb_count(c, ch[i]) <= 3)) continue;
                float area = lb_half_area(box[i]);
                if (LBVH_OPEN_SMALL == 2 && lb_count(c, ch[i]) <= 3) {
                    // SAH gain of splitting a small leaf: A*n - (Al*nl + Ar*nr), in triangle-test units
                    LbBox bl, br;
                    lb_child_box(c, c.left[ch[i]], &bl);
                    lb_child_box(c, c.right[ch[i]], &br);
                    area = area * (float)lb_count(c, ch[i]) - (lb_half_area(bl) * (float)lb_count(c, c.left[ch[i]]) +
                                                                lb_half_area(br) * (float)lb_count(c, c.right[ch[i]]));
                }
                if (area > bestArea) {
                    bestArea = area;
                    best = i;
                }
            }
            if (best < 0) break;
            const int32_t open = ch[best];
            ch[best] = c.left[open];
            lb_child_box(c, ch[best], &box[best]);
            ch[k] = c.right[open];
            lb_child_box(c, ch[k], &box[k]);
            ++k;
        }
    }
    // A subtree of 2-3 triangles that found no free slots is either a leaf child (every ray entering its box tests
    // all its triangles: A*n) or a small wide node of its own (A for the node + the triangles' own boxes).
    uint8_t ntri[W];
    for (int i = 0; i < k; ++i) {
        const int32_t cnt = lb_count(c, ch[i]);
        bool isLeaf = ch[i] < 0;
        if (ch[i] >= 0 && cnt <= 3) {
            float triAreas = 0.f;
            for (int32_t t = 0; t < cnt; ++t) {
                LbBox tb;
                lb_tri_box(c.vertices + 9 * (int64_t)c.sorted[c.first[ch[i]] + t], &tb);
                triAreas += lb_half_area(tb);
            }
            const float A = lb_half_area(box[i]);
            isLeaf = LBVH_OPEN_SMALL == 0 || A * (float)cnt <= A + triAreas;
        }
        ntri[i] = isLeaf ? (uint8_t)cnt : 0;
    }
    // octant-ordered slots + quantisation, identical to the host builder (wbvh.h)
    WbBox wb[W];
    for (int i = 0; i < k; ++i)
        for (int a = 0; a < 3; ++a) {
            wb[i].lo[a] = box[i].lo[a];
            wb[i].hi[a] = box[i].hi[a];
        }
    int childAt[W];
    wbvh_assign_slots(wb, k, childAt);
    // allocation: inner children contiguous in slot order, leaf triangles contiguous in slot order
    uint32_t nInner = 0, nTri = 0;
    for (int s = 0; s < W; ++s) {
        const int i = childAt[s];
        if (i < 0) continue;
        if (ntri[i])
            nTri += (uint32_t)ntri[i];
        else
            ++nInner;
    }
    const uint32_t childBase = nInner ? lb_atomic_add(c.n_nodes, nInner) : 0u;
    const uint32_t triBase = nTri ? lb_atomic_add(c.n_tris, nTri) : 0u;
    const uint32_t qBase = nInner ? lb_atomic_add(c.q_out_count, nInner) : 0u;

    WbvhNode node;
    wbvh_encode_node(wb, childAt, ntri, c.cell_floor, &node);
    node.child_base = childBase;
    uint32_t triOffset = 0, innerRank = 0;
    for (int s = 0; s < W; ++s) {
        const int i = childAt[s];
        if (i < 0) continue;
        const int32_t cnt = lb_count(c, ch[i]);
        if (ntri[i]) {
            const int64_t f0 = ch[i] < 0 ? (int64_t)(~ch[i]) : (int64_t)c.first[ch[i]];
            for (int32_t t = 0; t < cnt; ++t) {
                const uint32_t tri = c.sorted[f0 + t];
                const uint32_t pos = triBase + triOffset + (uint32_t)t;
                const float *v = c.vertices + 9 * (int64_t)tri;
                TriRecord r;
                for (int a = 0; a < 3; ++a) {
                    r.p0[a] = v[a];
                    r.p1[a] = v[3 + a];
                    r.p2[a] = v[6 + a];
                }
                const uint8_t vf = c.vertex_flags ? c.vertex_flags[tri] : 3;
                r.prim = tri;
                r.mat_flags = (uint32_t)(c.material_id ? c.material_id[tri] : 0) | ((c.flip && c.flip[tri]) ? B200PT_TRI_FLIP : 0u) |
                              ((c.has_normals && (vf & 1)) ? B200PT_TRI_HAS_NORMALS : 0u) |
                              ((c.has_uvs && (vf & 2)) ? B200PT_TRI_HAS_UVS : 0u);
                r.light = c.light_id ? c.light_id[tri] : -1;
                c.tris[pos] = r;
                c.prim_to_tri[tri] = pos;
            }
            triOffset += (uint32_t)cnt;
        } else {
            LbvhItem next;
            next.node2 = ch[i];
            next.wide = childBase + innerRank;
            c.q_out[qBase + innerRank] = next;
            ++innerRank;
        }
    }
    if (it.wide < c.node_cap) {
        memcpy(&c.nodes[it.wide], &node, sizeof(node));  // as bytes: an assignment costs k_lbvh_collapse 4 registers
        c.tri_base[it.wide] = triBase;
    }
}

// ---- 6. triangles that never enter the tree still need records (an area light may sit on one)
B200_HD void lbvh_leftover(const LbvhCtx &c, int64_t i) {
    if (c.prim_to_tri[i] != 0xffffffffu) return;
    const uint32_t pos = lb_atomic_add(c.n_tris, 1u);
    const float *v = c.vertices + 9 * i;
    TriRecord r;
    for (int a = 0; a < 3; ++a) {
        r.p0[a] = v[a];
        r.p1[a] = v[3 + a];
        r.p2[a] = v[6 + a];
    }
    const uint8_t vf = c.vertex_flags ? c.vertex_flags[i] : 3;
    r.prim = (uint32_t)i;
    r.mat_flags = (uint32_t)(c.material_id ? c.material_id[i] : 0) | ((c.flip && c.flip[i]) ? B200PT_TRI_FLIP : 0u) |
                  B200PT_TRI_DEGENERATE | ((c.has_normals && (vf & 1)) ? B200PT_TRI_HAS_NORMALS : 0u) |
                  ((c.has_uvs && (vf & 2)) ? B200PT_TRI_HAS_UVS : 0u);
    r.light = c.light_id ? c.light_id[i] : -1;
    c.tris[pos] = r;
    c.prim_to_tri[i] = pos;
}

}  // namespace b200pt
#endif
