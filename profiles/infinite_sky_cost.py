"""What an environment map costs on the benchmark scene: cfg4's 10 M-triangle soup with its 16 area lights at 1920x1080,
rendered with and without a seeded 2048x1024 sky (an InfiniteAreaLight with "string mapname"; its Distribution2D is
4096x2048), alternating the two in one process.  The sky's tables are the ones the reference builds: pbrt_b200 renders
a small scene with the same map and hands them over through B200PT_DUMP_SCENE.  Prints one JSON line.

  python profiles/infinite_sky_cost.py [--spp 64] [--rounds 2] [--steps 3] [--profile]     # on the GPU box

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


def sky_map(seed=2048, w=2048, h=1024):
    """A smooth sky with a sun: a vertical gradient, low-frequency noise and one bright disc."""
    rng = np.random.default_rng(seed)
    v = (np.arange(h) + 0.5) / h
    u = (np.arange(w) + 0.5) / w
    base = np.clip(1.2 - v, 0.05, None)[:, None, None] * np.array([0.6, 0.75, 1.0], np.float32)
    noise = rng.uniform(0.8, 1.2, (h // 64, w // 64, 3)).repeat(64, 0).repeat(64, 1)
    img = (base * noise).astype(np.float32)
    du, dv = np.meshgrid(u - 0.3, v - 0.25)
    img[du * du + dv * dv < 0.0004] = (400.0, 380.0, 350.0)
    return img


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    pkg = graft.load_package()
    from pbrt_v3_distributed_b200 import abi, scenes
    tmp = tempfile.mkdtemp(prefix="b200pt_sky_")
    # the host's tables of the sky: a small scene with the same light through the drop-in binary
    sky = sky_map()
    small = scenes.SceneArrays(1000, materials=("matte",), soup_version=1, n_lights=16, infinite_lights=[dict(map=sky)])
    path = scenes.write_pbrt(tmp, "sky", small, 16, 16, 1)
    dump = os.path.join(tmp, "sky.dump")
    subprocess.run([PLUGIN, "--quiet", "--outfile", os.path.join(tmp, "sky_small.pfm"), os.path.basename(path)], cwd=tmp,
                   env=dict(os.environ, B200PT_DUMP_SCENE=dump), check=True, capture_output=True)
    (light, tables), = scenes.read_dump_infinite(dump, abi).items()

    n_tris, mats, w, h = 10000000, ("matte", "glass", "metal", "plastic"), 1920, 1080
    setup = scenes.RenderSetup(w, h, args.spp, max_depth=5)
    ctx = pkg.Context(0)
    arms = {}
    t0 = time.time()
    for name, inf in (("no_sky", ()), ("sky", (dict(map=sky),))):
        arr = scenes.SceneArrays(n_tris, materials=mats, soup_version=1, n_lights=16, infinite_lights=inf)
        scene = pkg.Scene(ctx, arr.desc(), keepalive=arr)
        if inf:
            assert light == arr.n_lights - 1
            scene.set_infinite_light(light, tables)
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
        for name in ("no_sky", "sky"):
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
           "sky_map": "2048x1024 (Distribution2D 4096x2048), seed 2048", "gpu": q.stdout.strip(), "scene_build_s": round(build_s, 1)}
    for name, a in arms.items():
        rates = [r / (ms * 1e3) for r, ms in zip(a["rays"], a["ms"])]
        out[name] = {"mrays_per_s_median": float(np.median(rates)), "mrays_per_s_min": min(rates), "mrays_per_s_max": max(rates),
                     "ms_median": float(np.median(a["ms"])), "rays_per_step": a["rays"][-1], "steps": len(rates)}
        if args.profile:  # device ms per step: closest-hit traversal, any-hit traversal, every other launch
            c = np.median(np.array(a["classes"][-len(rates):]), axis=0)
            out[name]["device_ms"] = {"closest": float(c[0]), "any": float(c[1]), "other": float(c[2])}
    out["sky_time_ratio"] = out["sky"]["ms_median"] / out["no_sky"]["ms_median"]
    print(json.dumps(out))
    for a in arms.values():
        a["scene"].close()
    ctx.close()


if __name__ == "__main__":
    main()
