"""What alpha masks cost on the benchmark scene: cfg4's 10 M-triangle soup with its 16 area lights at 1920x1080, rendered
without masks and with a seeded 2048x2048 alpha mask (repeat wrap, about half of its texels exactly 0) on every matte
triangle, the two arms alternating step by step in one process.  The soup has no uvs, so every masked triangle maps
GetUVs' defaults (0,0), (1,0), (1,1) onto the mask.  Prints one JSON line with the card's name and power limit.

  python profiles/alpha_cost.py [--spp 64] [--steps 6] [--profile]     # on the GPU box

Rays are the library's own counters (regular + shadow ray intersection tests); time is the host clock around
render_tiles + synchronize of all tiles.  Scene builds are excluded.  --profile brackets every launch with CUDA events
(render option "profile") and adds the device time per traversal launch; take the rates from a run without it."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402


def alpha_map(seed=2048, n=2048):
    """Blocks of 8 texels, each 0 with probability 1/2, else in [0.05, 1)."""
    rng = np.random.default_rng(seed)
    keep = rng.uniform(size=(n // 8, n // 8)) < 0.5
    vals = rng.uniform(0.05, 1.0, (n, n)).astype(np.float32)
    return np.where(keep.repeat(8, 0).repeat(8, 1), vals, np.float32(0)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    pkg = graft.load_package()
    from pbrt_v3_distributed_b200 import abi, scenes
    n_tris, mats, w, h = 10000000, ("matte", "glass", "metal", "plastic"), 1920, 1080
    setup = scenes.RenderSetup(w, h, args.spp, max_depth=5)
    ctx = pkg.Context(0)
    mask = alpha_map()
    arms = {}
    t0 = time.time()
    for name in ("unmasked", "masked"):
        arr = scenes.SceneArrays(n_tris, materials=mats, soup_version=1, n_lights=16)
        scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
        if name == "masked":
            mid = scene.add_alpha_mask(mask, abi.WRAP_REPEAT)
            scene.set_alpha_masks(np.where(arr.material_id == arr.material_names.index("matte"), mid, -1).astype(np.int32), None)
        r = pkg.Render(scene, setup)
        if args.profile:
            r.set_option("profile", 1)
        arms[name] = {"scene": scene, "arr": arr, "render": r, "ms": [], "rays": [], "per_launch": []}
    build_s = time.time() - t0

    def step(a):
        r = a["render"]
        r.clear()
        r.reset_stats()
        ctx.synchronize()
        t = time.time()
        r.render_tiles()
        ctx.synchronize()
        dt = time.time() - t
        st = r.stats()
        if args.profile:
            a["per_launch"].append((st["closest_ms"] / max(1, st["closest_launches"]), st["any_ms"] / max(1, st["any_launches"])))
        return dt, st["regular_rays"] + st["shadow_rays"]

    for a in arms.values():
        step(a)  # warm-up
        a["per_launch"].clear()
    for _ in range(args.steps):
        for a in arms.values():
            dt, rays = step(a)
            a["ms"].append(1e3 * dt)
            a["rays"].append(rays)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"workload": "cfg4 scene (10M triangles, 16 area lights, 4 BSDF families), %dx%d, %d spp, maxdepth 5, uniform" % (w, h, args.spp),
           "mask": "2048x2048 alpha, repeat, ~half of the texels 0 in 8x8 blocks, seed 2048, on every matte triangle",
           "gpu": q.stdout.strip(), "scene_build_s": round(build_s, 1)}
    for name, a in arms.items():
        rates = [r / (ms * 1e3) for r, ms in zip(a["rays"], a["ms"])]
        out[name] = {"mrays_per_s_median": float(np.median(rates)), "mrays_per_s_min": min(rates), "mrays_per_s_max": max(rates),
                     "ms_median": float(np.median(a["ms"])), "rays_per_step": a["rays"][-1], "steps": len(rates)}
        if args.profile:  # device ms per traversal launch (median over the steps): closest hit, any hit
            c = np.median(np.array(a["per_launch"]), axis=0)
            out[name]["device_ms_per_launch"] = {"closest": float(c[0]), "any": float(c[1])}
    out["mask_time_ratio"] = out["masked"]["ms_median"] / out["unmasked"]["ms_median"]
    print(json.dumps(out))
    for a in arms.values():
        a["render"].close()
        a["scene"].close()
    ctx.close()


if __name__ == "__main__":
    main()
