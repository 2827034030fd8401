"""What image textures cost on the benchmark scene: cfg4's 10 M-triangle soup with its 16 area lights at 1920x1080,
rendered with constant materials and with a seeded 2048x2048 imagemap (EWA, repeat wrap) on each BSDF family's main
spectrum parameter (matte Kd, plastic Kd, metal k, glass Kt), alternating the two in one process.  The MIPMap is the one
the reference builds: pbrt_b200 renders a small scene with the same texture and hands its pyramid over through
B200PT_DUMP_SCENE.  Prints one JSON line with the card's name and power limit.

  python profiles/texture_cost.py [--spp 64] [--rounds 2] [--steps 3] [--profile]     # on the GPU box

Rays are the library's own counters (regular + shadow ray intersection tests); time is the host clock around
render_tiles + synchronize of all tiles.  Scene builds are excluded.  --profile brackets every launch with CUDA events
(render option "profile") and adds the device time per kernel class; take the rates from a run without it."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

PLUGIN = os.path.join(ROOT, "oracle", "_ref", "plugin", "pbrt_b200")


def texture_map(seed=2048, n=2048):
    """Texels in [0.05, 0.95): blocks of 16 texels over fine noise."""
    rng = np.random.default_rng(seed)
    blocks = rng.uniform(0.1, 0.9, (n // 16, n // 16, 3)).repeat(16, 0).repeat(16, 1)
    return np.clip(blocks + rng.uniform(-0.05, 0.05, (n, n, 3)), 0.05, 0.95).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    pkg = graft.load_package()
    from pbrt_v3_distributed_b200 import abi, scenes
    tmp = tempfile.mkdtemp(prefix="b200pt_tex_")
    # the host's MIPMap of the texture: a small scene with the same map through the drop-in binary
    tex = texture_map()
    small = scenes.SceneArrays(1000, materials=("matte",), soup_version=1, n_lights=16, textures={"matte": {"Kd": dict(map=tex)}})
    path = scenes.write_pbrt(tmp, "tex", small, 16, 16, 1)
    dump = os.path.join(tmp, "tex.dump")
    subprocess.run([PLUGIN, "--quiet", "--outfile", os.path.join(tmp, "tex_small.pfm"), os.path.basename(path)], cwd=tmp,
                   env=dict(os.environ, B200PT_DUMP_SCENE=dump), check=True, capture_output=True)
    (mip,), _ = scenes.read_dump_textures(dump, abi)

    n_tris, mats, w, h = 10000000, ("matte", "glass", "metal", "plastic"), 1920, 1080
    setup = scenes.RenderSetup(w, h, args.spp, max_depth=5)
    ctx = pkg.Context(0)
    arms = {}
    t0 = time.time()
    slots = {"matte": abi.TEX_KD, "plastic": abi.TEX_KD, "metal": abi.TEX_K, "glass": abi.TEX_KT}
    for name in ("constant", "textured"):
        arr = scenes.SceneArrays(n_tris, materials=mats, soup_version=1, n_lights=16)
        scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
        if name == "textured":
            mid = scene.add_mipmap(mip["levels"], mip["wrap"], mip["trilinear"], mip["max_anisotropy"], mip["weight_lut"])
            for m in mats:
                scene.bind_texture(arr.material_names.index(m), slots[m], mid)
        arms[name] = {"scene": scene, "arr": arr, "ms": [], "rays": [], "classes": []}
    build_s = time.time() - t0

    def step(arm, r):
        r.clear()
        r.reset_stats()
        ctx.synchronize()
        t = time.time()
        r.render_tiles()
        ctx.synchronize()
        dt = time.time() - t
        st = r.stats()
        arm["classes"].append((st["closest_ms"], st["any_ms"], st["shade_ms"]))
        return dt, st["regular_rays"] + st["shadow_rays"]

    for rnd in range(args.rounds):
        for name in ("constant", "textured"):
            a = arms[name]
            r = pkg.Render(a["scene"], setup)
            if args.profile:
                r.set_option("profile", 1)
            step(a, r)  # warm-up
            for _ in range(args.steps):
                dt, rays = step(a, r)
                a["ms"].append(1e3 * dt)
                a["rays"].append(rays)
            r.close()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"workload": "cfg4 scene (10M triangles, 16 area lights, 4 BSDF families), %dx%d, %d spp, maxdepth 5, uniform" % (w, h, args.spp),
           "texture": "2048x2048 imagemap, EWA, repeat, seed 2048, on matte Kd, plastic Kd, metal k, glass Kt", "gpu": q.stdout.strip(), "scene_build_s": round(build_s, 1)}
    for name, a in arms.items():
        rates = [r / (ms * 1e3) for r, ms in zip(a["rays"], a["ms"])]
        out[name] = {"mrays_per_s_median": float(np.median(rates)), "mrays_per_s_min": min(rates), "mrays_per_s_max": max(rates),
                     "ms_median": float(np.median(a["ms"])), "rays_per_step": a["rays"][-1], "steps": len(rates)}
        if args.profile:  # device ms per step: closest-hit traversal, any-hit traversal, every other launch
            c = np.median(np.array(a["classes"][-len(rates):]), axis=0)
            out[name]["device_ms"] = {"closest": float(c[0]), "any": float(c[1]), "other": float(c[2])}
    out["texture_time_ratio"] = out["textured"]["ms_median"] / out["constant"]["ms_median"]
    print(json.dumps(out))
    for a in arms.values():
        a["scene"].close()
    ctx.close()


if __name__ == "__main__":
    main()
