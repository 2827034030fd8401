"""Round-2 knob sweep on one scene build: times a few wavefront batches of a workload for each k_trace setting
(b200pt_render_set_option: refill_lanes, postpone_pct, overlap).  Device time per kernel class comes
from the library's own CUDA events ("profile"); rays are the reference's counters.

  python profiles/sweep2.py [workload] [n_batches] [setting ...]     setting = name=value[,name=value...]
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402
import bench  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "cfg3"
n_batches = int(sys.argv[2]) if len(sys.argv) > 2 else 3
settings = sys.argv[3:] or ["", "refill_lanes=22", "refill_lanes=28", "postpone_pct=25", "postpone_pct=60", "overlap=0"]
pkg = graft.load_package()
from pbrt_v3_distributed_b200 import scenes  # noqa: E402

n_tris, mats, xres, yres, spp, depth, n_lights, _ = bench.WORKLOADS[name]
t0 = time.time()
arr = scenes.SceneArrays(n_tris, materials=mats, soup_version=1, n_lights=n_lights, **bench.workload_scene_kwargs(name))
gen_s = time.time() - t0
setup = scenes.RenderSetup(xres, yres, spp, max_depth=depth)
ctx = pkg.Context(0)
t0 = time.time()
scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
build_s = time.time() - t0
info = scene.info()
print("%s: scene arrays %.1f s, scene_create %.1f s, %d nodes (%.0f MB nodes, %.0f MB triangles)" %
      (name, gen_s, build_s, info["n_nodes"], info["node_bytes"] / 1e6, info["tri_bytes"] / 1e6), flush=True)
r = pkg.Render(scene, setup)
per_batch = max(1, int(os.environ.get("B200PT_BATCH_PATHS", 16 << 20)) // (256 * spp))
mid = (r.tiles_y // 2) * r.tiles_x + r.tiles_x // 4
tiles = (mid + np.arange(per_batch * n_batches)) % r.n_tiles
defaults = dict(refill_lanes=26, postpone_pct=40, overlap=1)
# instrumented pass once: nodes / triangles per ray
r.set_option("instrument", 1)
r.render_tiles(tiles[:per_batch])
ctx.synchronize()
st = r.stats()
print("instrumented: %.2f nodes/ray %.2f tris/ray (closest), %.2f / %.2f (any-hit), stack overflows %d" %
      (st["nodes_visited"] / max(st["regular_rays"], 1), st["tris_tested"] / max(st["regular_rays"], 1),
       st["any_nodes_visited"] / max(st["shadow_rays"], 1), st["any_tris_tested"] / max(st["shadow_rays"], 1),
       st["stack_overflows"]), flush=True)
r.set_option("instrument", 0)
for s in settings:
    opts = dict(defaults)
    for kv in filter(None, s.split(",")):
        k, v = kv.split("=")
        opts[k] = int(v)
    for k, v in opts.items():
        r.set_option(k, v)
    r.render_tiles(tiles[:per_batch])  # warm-up
    ctx.synchronize()
    r.reset_stats()
    r.set_option("profile", 1)
    t0 = time.time()
    r.render_tiles(tiles)
    ctx.synchronize()
    wall = time.time() - t0
    st = r.stats()
    r.set_option("profile", 0)
    rays = st["regular_rays"] + st["shadow_rays"]
    print("%-32s %7.1f Mrays/s wall (%7.1f ms); closest %7.1f ms (%6.1f Mrays/s), any %6.1f ms (%6.1f Mrays/s), other %6.1f ms" %
          (s or "default", rays / wall / 1e6, wall * 1e3, st["closest_ms"], st["regular_rays"] / max(st["closest_ms"], 1e-9) / 1e3,
           st["any_ms"], st["shadow_rays"] / max(st["any_ms"], 1e-9) / 1e3, st["shade_ms"]), flush=True)
