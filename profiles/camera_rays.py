"""Camera-ray share of cfg4's traversal time.  Renders the same middle-of-film tiles as sweep2.py twice: at max_depth=0,
where only camera rays are traced and they run alone on the main stream (so `closest_ms` is camera-ray traversal and
nothing else), and at the workload's full depth.  Device times come from the library's own CUDA events ("profile").

  python profiles/camera_rays.py [workload] [n_batches] [repeats]

Set B200PT_LIB_VARIANT to time an experimental build of the library (see csrc/Makefile).
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402
import bench  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "cfg4"
n_batches = int(sys.argv[2]) if len(sys.argv) > 2 else 4
repeats = int(sys.argv[3]) if len(sys.argv) > 3 else 3
pkg = graft.load_package()
from pbrt_v3_distributed_b200 import scenes  # noqa: E402

n_tris, mats, xres, yres, spp, depth, n_lights, _ = bench.WORKLOADS[name]
arr = scenes.SceneArrays(n_tris, materials=mats, soup_version=1, n_lights=n_lights, **bench.workload_scene_kwargs(name))
ctx = pkg.Context(0)
scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
print("%s: library %s" % (name, os.environ.get("B200PT_LIB_VARIANT") or "default"), flush=True)


def run(max_depth):
    r = pkg.Render(scene, scenes.RenderSetup(xres, yres, spp, max_depth=max_depth))
    # n_batches batches of 32 Mi path slots (the library renders them in batches of its own size, api.cu)
    per_batch = max(1, (32 << 20) // (256 * spp))
    mid = (r.tiles_y // 2) * r.tiles_x + r.tiles_x // 4
    tiles = (mid + np.arange(per_batch * n_batches)) % r.n_tiles
    r.set_option("instrument", 1)
    r.render_tiles(tiles[:per_batch])
    ctx.synchronize()
    st = r.stats()
    nodes = st["nodes_visited"] / max(st["regular_rays"], 1)
    tris = st["tris_tested"] / max(st["regular_rays"], 1)
    overflows = st["stack_overflows"]
    r.set_option("instrument", 0)
    r.render_tiles(tiles[:per_batch])  # warm-up
    ctx.synchronize()
    for k in range(repeats):
        r.reset_stats()
        r.set_option("profile", 1)
        t0 = time.time()
        r.render_tiles(tiles)
        ctx.synchronize()
        wall = time.time() - t0
        st = r.stats()
        r.set_option("profile", 0)
        print("max_depth=%d run %d: %d tiles, wall %.1f ms, closest %.1f ms, any %.1f ms, other %.1f ms; %d camera rays "
              "(%.1f Mrays/s over closest_ms), %d regular, %d shadow; %.2f nodes / %.2f tris per closest-hit ray, "
              "%d stack overflows" %
              (max_depth, k, len(tiles), wall * 1e3, st["closest_ms"], st["any_ms"], st["shade_ms"], st["camera_rays"],
               st["camera_rays"] / max(st["closest_ms"], 1e-9) / 1e3, st["regular_rays"], st["shadow_rays"], nodes, tris,
               overflows), flush=True)
    r.close()


run(0)
run(depth)
