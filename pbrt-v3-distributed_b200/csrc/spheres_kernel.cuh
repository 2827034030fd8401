// spheres_kernel.cuh -- included twice by kernels.cu: once as the kernel scenes without alpha masks launch (B200PT_WALK(x) = x,
// B200PT_WALK_ALPHA(off) empty), once as its twin for scenes with masks (x##_alpha, the AlphaTest of the launch for the
// tree whose triangles start at `off`).  No include guard on purpose.
// All instances against one ray, as a resumable state machine: through the tree over their leaf boxes when there is
// one (its leaf "triangles" carry instance numbers), else one by one.  Each lane walks the tree over the instances'
// boxes, picks the next candidate instance, or takes ONE step inside that instance's tree per call of step(), so that
// the lanes of a warp meet again after every step instead of after whole nested traversals (measured with nested loops:
// 2.4 of 32 lanes active per instruction) and a lane whose ray is done can take the next ray (k_spheres).
template <bool ANY_HIT>
struct B200PT_WALK(InstanceWalk) {
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
            if (!(T2.cur_y & 0xff000000u) || trav_step<ANY_HIT, false>(T2, R2, S2, bn, bb, bt, a.lut, &ctr B200PT_WALK_ALPHA(cur_tri_off))) {
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
template <bool ANY_HIT, bool CLASSIFY>
__global__ void __launch_bounds__(128) B200PT_WALK(k_spheres)(const TraceArgs a) {
    const uint32_t n = *a.count;
#ifndef B200PT_HOST_EMU
    const int lane = threadIdx.x & 31;
#endif
    B200PT_WALK(InstanceWalk)<ANY_HIT> W;
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
        // ---- converged: idle lanes fetch new rays, test the spheres, set up the walk over the instances
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
