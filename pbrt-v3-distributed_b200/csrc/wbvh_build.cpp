// wbvh_build.cpp -- host builder of the 7-wide compressed BVH (see wbvh.h).
//
// Replaces BVHAccel's constructor (accelerators/bvh.cpp:183-225: SAH
// recursiveBuild :236-402, flattenBVHTree :640-658).  The tree topology is
// not part of the parity contract -- closest hits are decided by the exact
// watertight triangle test and are topology independent (DESIGN.md,
// "Traversal order and ties") -- so the build is designed for the GPU
// traversal kernel, not to mimic the reference's binary tree:
//   1. binary BVH by binned SAH (16 bins) down to single triangles, built
//      top-down with one std::thread per large subtree;
//   2. SAH-optimal collapse to 7 children per node (dynamic programme of
//      Ylitie et al. 2017, section 3.1; leaves of <= 3 triangles);
//   3. children placed in octant-ordered slots (wbvh_assign_slots) so that
//      visiting slots by (slot XOR ray octant) approximates front-to-back order;
//   4. child boxes quantised to 8 bits per coordinate on a power-of-two grid
//      anchored at the node's min corner, rounded outward in exact arithmetic
//      (wbvh_encode_node); the traversal kernel decodes the bytes exactly and
//      adds its own fraction-of-a-cell slack for float rounding.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <thread>

#include "wbvh.h"

namespace b200pt {
namespace {

struct Box {
    float lo[3], hi[3];
    void reset() {
        for (int a = 0; a < 3; ++a) {
            lo[a] = INFINITY;
            hi[a] = -INFINITY;
        }
    }
    void grow(const Box &b) {
        for (int a = 0; a < 3; ++a) {
            lo[a] = std::min(lo[a], b.lo[a]);
            hi[a] = std::max(hi[a], b.hi[a]);
        }
    }
    void grow(const float *p) {
        for (int a = 0; a < 3; ++a) {
            lo[a] = std::min(lo[a], p[a]);
            hi[a] = std::max(hi[a], p[a]);
        }
    }
    float half_area() const {
        float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        if (!(dx >= 0) || !(dy >= 0) || !(dz >= 0)) return 0.f;
        return dx * dy + dy * dz + dz * dx;
    }
};

struct Node2 {
    Box box;
    int32_t left, right;   // children (inner) or -1
    int32_t first, count;  // leaf range in idx[] (count > 0 <=> binary leaf = one triangle)
    int32_t ntri;          // triangles in the subtree: idx[first .. first + ntri)
};

struct Builder2 {
    const Box *tbox;
    const float *cent;  // 3 per triangle
    std::vector<int32_t> idx;
    std::vector<Node2> nodes;
    std::atomic<int32_t> next_node{0};
    std::atomic<int> threads_free{0};

    int32_t alloc() { return next_node.fetch_add(1); }

    void build(int32_t node, int32_t first, int32_t count) {
        Node2 &n = nodes[node];
        Box b, cb;
        b.reset();
        cb.reset();
        for (int32_t i = first; i < first + count; ++i) {
            b.grow(tbox[idx[i]]);
            cb.grow(cent + 3 * (size_t)idx[i]);
        }
        n.box = b;
        n.left = n.right = -1;
        n.first = first;
        n.count = 0;
        n.ntri = count;
        if (count == 1) {
            n.count = 1;
            return;
        }
        // binned SAH over the centroid bounds
        const int NB = 16;
        int bestAxis = -1, bestBin = -1;
        float bestCost = INFINITY;
        for (int axis = 0; axis < 3; ++axis) {
            float c0 = cb.lo[axis], c1 = cb.hi[axis];
            if (!(c1 > c0)) continue;
            float scale = NB / (c1 - c0);
            Box bb[NB];
            int bc[NB];
            for (int i = 0; i < NB; ++i) {
                bb[i].reset();
                bc[i] = 0;
            }
            for (int32_t i = first; i < first + count; ++i) {
                int t = idx[i];
                int bi = std::min(NB - 1, std::max(0, (int)((cent[3 * (size_t)t + axis] - c0) * scale)));
                bb[bi].grow(tbox[t]);
                bc[bi]++;
            }
            float rightArea[NB];
            int rightCount[NB];
            Box acc;
            acc.reset();
            int cnt = 0;
            for (int i = NB - 1; i > 0; --i) {
                acc.grow(bb[i]);
                cnt += bc[i];
                rightArea[i] = acc.half_area();
                rightCount[i] = cnt;
            }
            acc.reset();
            cnt = 0;
            for (int i = 0; i < NB - 1; ++i) {
                acc.grow(bb[i]);
                cnt += bc[i];
                if (cnt == 0 || rightCount[i + 1] == 0) continue;
                float cost = acc.half_area() * cnt + rightArea[i + 1] * rightCount[i + 1];
                if (cost < bestCost) {
                    bestCost = cost;
                    bestAxis = axis;
                    bestBin = i;
                }
            }
        }
        int32_t mid;
        if (bestAxis >= 0) {
            float c0 = cb.lo[bestAxis], scale = NB / (cb.hi[bestAxis] - c0);
            const float *cc = cent;
            int ax = bestAxis, bbn = bestBin;
            auto it = std::partition(idx.begin() + first, idx.begin() + first + count, [=](int32_t t) {
                int bi = std::min(NB - 1, std::max(0, (int)((cc[3 * (size_t)t + ax] - c0) * scale)));
                return bi <= bbn;
            });
            mid = (int32_t)(it - idx.begin());
        } else {
            mid = first + count / 2;  // all centroids coincide: split the range in half
        }
        if (mid == first || mid == first + count) mid = first + count / 2;
        int32_t l = alloc(), r = alloc();
        nodes[node].left = l;
        nodes[node].right = r;
        int32_t lc = mid - first, rc = count - lc;
        if (count > 65536 && threads_free.fetch_sub(1) > 0) {
            std::thread th([this, l, first, lc]() { build(l, first, lc); });
            build(r, mid, rc);
            th.join();
            threads_free.fetch_add(1);
        } else {
            if (count > 65536) threads_free.fetch_add(1);
            build(l, first, lc);
            build(r, mid, rc);
        }
    }
};

struct Child {
    int32_t node2;  // binary node
    Box box;
};

}  // namespace

void build_wbvh(const float *vertices, int64_t n_tris, const int32_t *material_id, const int32_t *light_id,
                const uint8_t *flip, const uint8_t *degenerate, int n_threads, Wbvh *out) {
    out->nodes.clear();
    out->tri_base.clear();
    out->tris.clear();
    out->prim_to_tri.assign((size_t)n_tris, 0xffffffffu);
    out->n_in_leaves = 0;
    out->max_depth = 0;

    std::vector<Box> tbox((size_t)n_tris);
    std::vector<float> cent(3 * (size_t)n_tris);
    Builder2 b2;
    b2.idx.reserve((size_t)n_tris);
    for (int64_t i = 0; i < n_tris; ++i) {
        Box b;
        b.reset();
        const float *v = vertices + 9 * i;
        b.grow(v);
        b.grow(v + 3);
        b.grow(v + 6);
        tbox[i] = b;
        bool finite = true;
        for (int a = 0; a < 3; ++a) {
            cent[3 * i + a] = 0.5f * b.lo[a] + 0.5f * b.hi[a];
            finite = finite && std::isfinite(b.lo[a]) && std::isfinite(b.hi[a]);
        }
        if (!(degenerate && degenerate[i]) && finite) b2.idx.push_back((int32_t)i);
    }
    auto make_tri = [&](int64_t i) {
        TriRecord t;
        const float *v = vertices + 9 * i;
        memcpy(t.p0, v, 12);
        memcpy(t.p1, v + 3, 12);
        memcpy(t.p2, v + 6, 12);
        t.prim = (uint32_t)i;
        t.mat_flags = (uint32_t)(material_id ? material_id[i] : 0) | ((flip && flip[i]) ? B200PT_TRI_FLIP : 0u) |
                      ((degenerate && degenerate[i]) ? B200PT_TRI_DEGENERATE : 0u);
        t.light = light_id ? light_id[i] : -1;
        return t;
    };
    const int32_t nLeafTris = (int32_t)b2.idx.size();
    out->tris.reserve((size_t)n_tris);

    if (nLeafTris > 0) {
        b2.tbox = tbox.data();
        b2.cent = cent.data();
        b2.nodes.resize(2 * (size_t)nLeafTris);
        b2.threads_free = std::max(0, n_threads - 1);
        int32_t root = b2.alloc();
        const bool trace = getenv("B200PT_BUILD_TRACE") != nullptr;
        auto tnow = []() { return std::chrono::steady_clock::now(); };
        auto tp0 = tnow();
        b2.build(root, 0, nLeafTris);
        auto tp1 = tnow();

        // ---- SAH-optimal collapse (Ylitie et al. 2017, section 3.1): cost[n][i-1] is the cheapest
        // way to represent the binary subtree n with at most i roots (i = 1..W-1); a single root is
        // either a leaf child (<= 3 triangles) or a W-wide node whose children come from
        // distributing the two binary children over W slots.
        constexpr int W = B200PT_WIDTH, R = W - 1;
        const int32_t nNodes2 = b2.next_node.load();
        float cNode = 1.0f, cPrim = 1.0f;  // a watertight triangle test costs about as many instructions as a node
        if (const char *e = getenv("B200PT_SAH_CNODE")) cNode = (float)atof(e);
        if (const char *e = getenv("B200PT_SAH_CPRIM")) cPrim = (float)atof(e);
        std::vector<float> cost((size_t)nNodes2 * R);
        std::vector<uint8_t> dec((size_t)nNodes2 * R);   // i=1: 0 leaf / 1 inner ; i>=2: 0 = reuse i-1, k = left gets k roots
        std::vector<uint8_t> splitW((size_t)nNodes2);    // left share when the node becomes a wide node
        for (int32_t n = nNodes2 - 1; n >= 0; --n) {
            const Node2 &nd = b2.nodes[n];
            float *c = &cost[(size_t)n * R];
            uint8_t *d = &dec[(size_t)n * R];
            const float A = nd.box.half_area();
            const float leafCost = nd.ntri <= 3 ? A * nd.ntri * cPrim : INFINITY;
            if (nd.count > 0) {  // single triangle
                for (int i = 0; i < R; ++i) {
                    c[i] = leafCost;
                    d[i] = 0;
                }
                splitW[n] = 0;
                continue;
            }
            const float *cl = &cost[(size_t)nd.left * R], *cr = &cost[(size_t)nd.right * R];
            auto distribute = [&](int j, int *bestK) {
                float best = INFINITY;
                *bestK = 1;
                for (int k = 1; k < j; ++k) {
                    if (k > R || j - k > R) continue;
                    float v = cl[k - 1] + cr[j - k - 1];
                    if (v < best) {
                        best = v;
                        *bestK = k;
                    }
                }
                return best;
            };
            int kW;
            const float innerCost = distribute(W, &kW) + A * cNode;
            splitW[n] = (uint8_t)kW;
            if (leafCost <= innerCost) {
                c[0] = leafCost;
                d[0] = 0;
            } else {
                c[0] = innerCost;
                d[0] = 1;
            }
            for (int i = 2; i <= R; ++i) {
                int k;
                float v = distribute(i, &k);
                if (v < c[i - 2]) {
                    c[i - 1] = v;
                    d[i - 1] = (uint8_t)k;
                } else {
                    c[i - 1] = c[i - 2];
                    d[i - 1] = 0;
                }
            }
        }
        auto tp2 = tnow();
        // children of a wide node: expand binary node `n` into at most `budget` roots
        struct Collector {
            const Builder2 &b2;
            const std::vector<uint8_t> &dec;
            Child *ch;
            int k;
            void collect(int32_t n, int budget) {
                const Node2 &nd = b2.nodes[n];
                int i = budget;
                while (i >= 2 && dec[(size_t)n * R + i - 1] == 0) --i;  // reuse the (i-1)-root solution
                if (i == 1 || nd.count > 0) {
                    ch[k++] = {n, nd.box};
                    return;
                }
                const int kl = dec[(size_t)n * R + i - 1];
                collect(nd.left, kl);
                collect(nd.right, i - kl);
            }
        };

        // ---- emit the wide nodes breadth-first so siblings are contiguous
        struct Pending {
            int32_t node2;
            uint32_t wide;
            int depth;
        };
        float absmax = 0.f;
        for (int a = 0; a < 3; ++a) {
            const Box &rb = b2.nodes[root].box;
            out->bounds_lo[a] = rb.lo[a];
            out->bounds_hi[a] = rb.hi[a];
            absmax = std::max(absmax, std::max(std::fabs(rb.lo[a]), std::fabs(rb.hi[a])));
        }
        const float cell_floor = B200PT_CELL_FLOOR * absmax;
        std::vector<Pending> queue;
        out->nodes.reserve((size_t)nLeafTris / 3 + 16);
        out->nodes.push_back(WbvhNode());
        queue.push_back({root, 0u, 1});
        for (size_t qi = 0; qi < queue.size(); ++qi) {
            Pending cur = queue[qi];
            out->max_depth = std::max(out->max_depth, cur.depth);
            Child ch[W];
            int k = 0;
            const Node2 &rn = b2.nodes[cur.node2];
            if (rn.count > 0 || (cur.node2 == root && dec[(size_t)root * R] == 0)) {
                ch[k++] = {cur.node2, rn.box};  // the whole scene is one leaf child of the root
            } else {
                Collector col{b2, dec, ch, 0};
                col.collect(rn.left, splitW[cur.node2]);
                col.collect(rn.right, W - splitW[cur.node2]);
                k = col.k;
            }
            WbBox box[W];
            uint8_t ntri[W];
            for (int i = 0; i < k; ++i) {
                memcpy(box[i].lo, ch[i].box.lo, 12);
                memcpy(box[i].hi, ch[i].box.hi, 12);
                const Node2 &c = b2.nodes[ch[i].node2];
                const bool isLeaf = c.count > 0 || dec[(size_t)ch[i].node2 * R] == 0;
                ntri[i] = isLeaf ? (uint8_t)c.ntri : 0;
            }
            int childAt[W];
            wbvh_assign_slots(box, k, childAt);
            WbvhNode node;
            memset(&node, 0, sizeof(node));
            wbvh_encode_node(box, childAt, ntri, cell_floor, &node);
            node.child_base = (uint32_t)out->nodes.size();
            const uint32_t triBase = (uint32_t)out->tris.size();
            for (int s = 0; s < W; ++s) {
                const int i = childAt[s];
                if (i < 0) continue;
                const Node2 &c = b2.nodes[ch[i].node2];
                if (ntri[i]) {
                    for (int t = 0; t < c.ntri; ++t) {
                        int32_t tri = b2.idx[c.first + t];
                        out->prim_to_tri[tri] = (uint32_t)out->tris.size();
                        out->tris.push_back(make_tri(tri));
                    }
                } else {
                    queue.push_back({ch[i].node2, (uint32_t)out->nodes.size(), cur.depth + 1});
                    out->nodes.push_back(WbvhNode());
                }
            }
            out->nodes[cur.wide] = node;
            if (out->tri_base.size() < out->nodes.size()) out->tri_base.resize(out->nodes.size(), 0u);
            out->tri_base[cur.wide] = triBase;
        }
        out->tri_base.resize(out->nodes.size(), 0u);
        out->n_in_leaves = (uint32_t)out->tris.size();
        if (trace)
            fprintf(stderr, "wbvh build: binary SAH %.3f s, collapse DP %.3f s, emit %.3f s\n",
                    std::chrono::duration<double>(tp1 - tp0).count(), std::chrono::duration<double>(tp2 - tp1).count(),
                    std::chrono::duration<double>(tnow() - tp2).count());
    } else {
        // empty scene: a root with no children
        WbvhNode node;
        memset(&node, 0, sizeof(node));
        const int none[B200PT_WIDTH] = {-1, -1, -1, -1, -1, -1, -1};
        wbvh_encode_node(nullptr, none, nullptr, 1.f, &node);
        out->nodes.push_back(node);
        out->tri_base.push_back(0u);
        out->max_depth = 1;
    }
    // triangles that can never be hit still need records (an area light may sit on one)
    for (int64_t i = 0; i < n_tris; ++i)
        if (out->prim_to_tri[i] == 0xffffffffu) {
            out->prim_to_tri[i] = (uint32_t)out->tris.size();
            out->tris.push_back(make_tri(i));
        }
}

int64_t validate_wbvh(const Wbvh &bvh) {
    int64_t bad = 0;
    if (bvh.tri_base.size() != bvh.nodes.size()) ++bad;
    // decoded slot boxes must contain what they refer to (p + q * cell is exact in double)
    struct BoxD {
        double lo[3], hi[3];
    };
    auto slot_box = [](const WbvhNode &n, int s) {
        BoxD b;
        for (int a = 0; a < 3; ++a) {
            const double c = wb_cell(n.e[a]);
            const int lo = a == 2 ? n.zq[s][0] : n.xyq[s][2 * a], hi = a == 2 ? n.zq[s][1] : n.xyq[s][2 * a + 1];
            b.lo[a] = (double)n.p[a] + lo * c;
            b.hi[a] = (double)n.p[a] + hi * c;
        }
        return b;
    };
    // true content bounds bottom-up (children have larger indices than their parents)
    std::vector<Box> content(bvh.nodes.size());
    for (int64_t ni = (int64_t)bvh.nodes.size() - 1; ni >= 0; --ni) {
        const WbvhNode &n = bvh.nodes[ni];
        Box cb;
        cb.reset();
        uint32_t inner = 0, triOff = 0;
        for (int s = 0; s < B200PT_WIDTH; ++s) {
            const int cnt = (n.lcount >> (2 * s)) & 3;
            const bool isInner = (n.imask >> s) & 1;
            if (isInner && cnt) ++bad;
            if (!isInner && !cnt) {
                if (n.xyq[s][0] != B200PT_EMPTY_LO || n.xyq[s][1] != 0 || n.xyq[s][2] != B200PT_EMPTY_LO || n.xyq[s][3] != 0 ||
                    n.zq[s][0] != B200PT_EMPTY_LO || n.zq[s][1] != 0)
                    ++bad;
                continue;
            }
            const BoxD sb = slot_box(n, s);
            Box got;
            got.reset();
            if (isInner) {
                uint32_t child = n.child_base + inner++;
                if (child >= bvh.nodes.size() || child <= (uint32_t)ni) {
                    ++bad;
                    continue;
                }
                got = content[child];
            } else {
                for (int t = 0; t < cnt; ++t) {
                    const size_t ti = (size_t)bvh.tri_base[ni] + triOff + t;
                    if (ti >= bvh.tris.size()) {
                        ++bad;
                        continue;
                    }
                    const TriRecord &tr = bvh.tris[ti];
                    got.grow(tr.p0);
                    got.grow(tr.p1);
                    got.grow(tr.p2);
                }
                triOff += cnt;
            }
            for (int a = 0; a < 3; ++a)
                if (!(sb.lo[a] <= (double)got.lo[a]) || !(sb.hi[a] >= (double)got.hi[a])) ++bad;
            cb.grow(got);
        }
        content[ni] = cb;
    }
    return bad;
}

}  // namespace b200pt
