// trace2_kernel.cuh -- included twice by kernels.cu: once as the kernel scenes without alpha masks launch (B200PT_WALK(x) = x,
// B200PT_WALK_ALPHA(off) empty), once as its twin for scenes with masks (x##_alpha, the AlphaTest of the launch for the
// tree whose triangles start at `off`).  No include guard on purpose.
template <bool ANY_HIT, bool CLASSIFY>
__global__ void __launch_bounds__(128, 6) B200PT_WALK(k_trace2)(const TraceArgs a) {
    __shared__ __align__(16) uint8_t s_lut[B200PT_LUT_BYTES];
    __shared__ float s_ray[B200PT_RAY_WORDS2 * 128];
    reinterpret_cast<uint4 *>(s_lut)[threadIdx.x] = __ldg(reinterpret_cast<const uint4 *>(a.lut) + threadIdx.x);
    __syncthreads();
    float *const my_ray = s_ray + threadIdx.x;
    const uint32_t n = *a.count;
    const int lane = threadIdx.x & 31;
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
        {
            int family = -1;
            if (fin) {
                const uint32_t best = __float_as_uint(my_ray[8 * 128]);
                if (ANY_HIT) {
                    slot_out(a.occ_out, slot, a.out_stride) = best != B200PT_MISS ? 1 : 0;
                } else {
                    if (a.hit_out) slot_out(a.hit_out, slot, a.out_stride) = best;
                    if (a.hit_inst_out && best != B200PT_MISS) slot_out(a.hit_inst_out, slot, a.out_stride) = __float_as_uint(my_ray[21 * 128]);
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
                if ((T.sp & B200PT_SP_OVERFLOW) && a.stats) atomicAdd(&a.stats[7], 1ull);
            }
            if (CLASSIFY) append_family(a.q_mat, a.qcount_mat, family, slot);
            fin = false;
        }
        // ---- converged: idle lanes fetch new rays
        {
            const bool want = !has && !exhausted;
            const uint32_t mask = __ballot_sync(FULL_MASK, want);
            if (mask) {
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
                    done = trav_tri_phase<ANY_HIT, false>(R, a.tri_base + noff, a.tris + (size_t)toff * 3, pend_x, pend_y, &ctr B200PT_WALK_ALPHA(toff));
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
