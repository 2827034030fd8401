"""Regenerates tests/golden/* from the UNMODIFIED reference (oracle/_ref/).

Run here (the container that has /root/reference):  python tests/golden/make_golden.py [render case ...]
Fixtures:
  sobol_tables.bin   generator matrices dumped from core/sobolmatrices.cpp (first 256 dims)
  probe.json         camera matrices, Sobol' sample streams, camera rays, material constants
                     (hex floats) from PerspectiveCamera / SobolSampler / MetalMaterial
  isect_*.npy        rays + BVHAccel::Intersect / IntersectP answers on a 3000-triangle soup
  render_*.pfm       pbrt_ref renders of small soup scenes (all four materials, uniform/power)
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

pkg = g.load_package()
ob = g.load_oracle()
from pbrt_v3_distributed_b200 import abi, scenes  # noqa: E402

CAMERAS = [(64, 64), (96, 64), (48, 80), (1024, 1024), (1920, 1080), (3840, 2160)]
sys.path.insert(0, os.path.dirname(HERE))
from render_cases import EXTRA, RENDERS  # noqa: E402

HALTON_CASES = [((0, 0, 700, 700), 8, 345, 678, 5, 0, 100), ((0, 0, 64, 48), 16, 3, 47, 15, 0, 120),
                ((0, 0, 1920, 1080), 1024, 1919, 1079, 1023, 0, 128), ((13, 7, 90, 50), 5, 13, 7, 0, 0, 64),
                ((0, 0, 100, 100), 3, 99, 0, 2, 0, 64), ((0, 0, 1, 1), 4, 0, 0, 3, 0, 16)]


def halton_fixtures():
    """HaltonSampler: the digit permutations of the first 128 prime bases and sample streams."""
    ob.probe("haltonperms", os.path.join(HERE, "halton_perms.bin"), 128)
    out = []
    for (bounds, spp, px, py, sample, dim0, n) in HALTON_CASES:
        vals = ob.probe("halton", *bounds, spp, px, py, sample, dim0, n).split()
        out.append({"bounds": bounds, "spp": spp, "px": px, "py": py, "sample": sample, "dim0": dim0,
                    "index": int(vals[0]), "values": vals[1:]})
    json.dump(out, open(os.path.join(HERE, "probe_halton.json"), "w"), indent=1)


FILTERS = {  # key: (probe args, the PixelFilter line of the .pbrt twin)
    "gaussian": (("gaussian", 2, 2, 2), 'PixelFilter "gaussian" "float xwidth" [2] "float ywidth" [2] "float alpha" [2]'),
    "gaussian_aniso": (("gaussian", 1.5, 2.5, 1), 'PixelFilter "gaussian" "float xwidth" [1.5] "float ywidth" [2.5] "float alpha" [1]'),
    "mitchell": (("mitchell", 2, 2), 'PixelFilter "mitchell" "float xwidth" [2] "float ywidth" [2]'),
    "triangle": (("triangle", 2, 2), 'PixelFilter "triangle" "float xwidth" [2] "float ywidth" [2]'),
    "sinc": (("sinc", 4, 4, 3), 'PixelFilter "sinc" "float xwidth" [4] "float ywidth" [4] "float tau" [3]'),
    "box1": (("box", 1, 1), 'PixelFilter "box" "float xwidth" [1] "float ywidth" [1]'),
}


def filter_fixtures():
    out = {}
    for key, (args, line) in FILTERS.items():
        txt = ob.probe("filtertable", *args).splitlines()
        out[key] = {"pbrt": line, "radius": txt[0].split()[1:], "table": txt[1:257]}
    json.dump(out, open(os.path.join(HERE, "filter_tables.json"), "w"), indent=0)


# "rgb" parameters of the spectral golden scenes (materials, area lights, sphere lights, point / spot / distant lights)
SPECTRAL_RGB = [(0.5, 0.5, 0.5), (0.0, 0.0, 0.0), (40.0, 40.0, 40.0), (60.0, 60.0, 60.0), (90.0, 90.0, 90.0), (6.0, 6.0, 6.0),
                (30.0, 24.0, 18.0), (0.8, 0.8, 0.8),
                (0.05, 0.08, 0.12), (0.3, 0.25, 0.2), (0.1, 0.05, 0.02), (0.15, 0.2, 0.3),  # sigma_a / sigma_s of the media
                # the remaining light intensities of tests/render_cases.py, so that every golden scene has 60-bin fixtures
                (3.14159265358979323846,) * 3, (3.14159265358979323846 / 4,) * 3, (9.0,) * 3, (400.0,) * 3, (80.0,) * 3,
                (150.0,) * 3, (1.0, 0.9, 0.8), (30.0,) * 3, (40.0,) * 3]
SPECTRAL_CONST = [0.25, 1.0, 0.9]                                      # float-default spectra (plastic, glass, mirror)
# rendered by the SampledSpectrum reference; instances + SampledSpectrum together are BASELINE configs[4]'s features
SPECTRAL_RENDERS = {"spectral_four": "four", "spectral_rough": "rough", "spectral_instances": "instances",
                    "spectral_spheres": "spheres", "spectral_delta_lights": "delta_lights"}
# VolPathIntegrator under the SampledSpectrum reference: golden name -> key of render_cases.VOLPATH
SPECTRAL_VOLPATH = {"spectral_volpath_fog": "volpath_fog", "spectral_volpath_fog_spheres": "volpath_fog_spheres"}


def spectral_fixtures():
    """Round-2 groundwork: the data liboracle_spectral.so needs from the SampledSpectrum build of the reference, and
    golden renders of that build (oracle/Makefile `ref_spectral`)."""
    import numpy as np
    f32 = np.float32

    def hx(v):
        return float(f32(v)).hex()
    args = [c for rgb in SPECTRAL_RGB for c in rgb]
    out = {"spectra": []}
    for line in ob.probe("spectral", *args, spectral=True).splitlines():
        tok = line.split()
        if tok[0] in ("cie_x", "cie_y", "cie_z"):
            out[tok[0]] = tok[1:]
        elif tok[0] == "rgb":
            out["spectra"].append([tok[1:4], tok[4:]])
        elif tok[0] == "copper_eta":
            out["spectra"].append([[hx(v) for v in scenes.COPPER_ETA], tok[1:]])
        elif tok[0] == "copper_k":
            out["spectra"].append([[hx(v) for v in scenes.COPPER_K], tok[1:]])
    for v in SPECTRAL_CONST:  # Spectrum(v): every bin holds v (spectrum.h:62-65)
        out["spectra"].append([[hx(v)] * 3, [hx(v)] * 60])
    json.dump(out, open(os.path.join(HERE, "spectral_tables.json"), "w"), indent=0)
    for gname, base in SPECTRAL_RENDERS.items():
        nt, mats, w, h, spp, depth, strat, nl = RENDERS[base]
        ex = EXTRA.get(base, {})
        arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
        path = scenes.write_pbrt("/tmp/golden_render", "render_" + gname, arr, w, h, spp, max_depth=depth, strategy=strat,
                                 **ex.get("camera", {}))
        ob.run_pbrt_ref(path, spectral=True)
        os.replace(os.path.join("/tmp/golden_render", "render_%s.pfm" % gname), os.path.join(HERE, "render_%s.pfm" % gname))
    from render_cases import VOLPATH
    for gname, vname in SPECTRAL_VOLPATH.items():
        base, medium, strat = VOLPATH[vname]
        nt, mats, w, h, spp, depth, _, nl = RENDERS[base]
        ex = EXTRA.get(base, {})
        arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
        path = scenes.write_pbrt("/tmp/golden_render", "render_" + gname, arr, w, h, spp, max_depth=depth, strategy=strat,
                                 integrator="volpath", medium=medium, **ex.get("camera", {}))
        ob.run_pbrt_ref(path, spectral=True)
        os.replace(os.path.join("/tmp/golden_render", "render_%s.pfm" % gname), os.path.join(HERE, "render_%s.pfm" % gname))


def volpath_goldens():
    """Images of the reference's VolPathIntegrator (tests/render_cases.py VOLPATH)."""
    from render_cases import VOLPATH
    for gname, (base, medium, strat) in VOLPATH.items():
        nt, mats, w, h, spp, depth, _, nl = RENDERS[base]
        ex = EXTRA.get(base, {})
        arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
        path = scenes.write_pbrt("/tmp/golden_render", "render_" + gname, arr, w, h, spp, max_depth=depth, strategy=strat,
                                 integrator="volpath", medium=medium, **ex.get("camera", {}))
        ob.run_pbrt_ref(path)
        os.replace(os.path.join("/tmp/golden_render", "render_%s.pfm" % gname), os.path.join(HERE, "render_%s.pfm" % gname))


def volpath_bounded_goldens():
    """The reference's volpath images of scenes with media bounded by null-material spheres (render_cases.VOLPATH_BOUNDED)."""
    from render_cases import VOLPATH_BOUNDED
    for gname, (fog, spheres) in VOLPATH_BOUNDED.items():
        arr = scenes.SceneArrays(3000, materials=("matte", "glass", "metal", "plastic"), soup_version=1, spheres=spheres)
        path = scenes.write_pbrt("/tmp/golden_render", "render_" + gname, arr, 40, 32, 8, max_depth=6, strategy="uniform",
                                 integrator="volpath", medium=fog)
        ob.run_pbrt_ref(path)
        os.replace(os.path.join("/tmp/golden_render", "render_%s.pfm" % gname), os.path.join(HERE, "render_%s.pfm" % gname))


def main():
    ob.probe("tables", os.path.join(HERE, "sobol_tables.bin"), 256)
    filter_fixtures()
    halton_fixtures()
    volpath_goldens()
    volpath_bounded_goldens()
    if os.path.exists(ob.PBRT_REF_SPECTRAL):
        spectral_fixtures()
    out = {"cameras": {}, "sobol": [], "camrays": []}
    cam_args = [0, 0, -4.5, 0, 0, 0, 0, 1, 0, 35]
    for (w, h) in CAMERAS:
        txt = ob.probe("camera", *cam_args, w, h).splitlines()
        rec = {}
        for line in txt:
            k, *v = line.split()
            rec[k] = v
        out["cameras"]["%dx%d" % (w, h)] = rec
    for (bounds, spp, px, py, sample, dim0, n) in [((0, 0, 64, 64), 16, 3, 5, 2, 0, 48),
                                                   ((0, 0, 1024, 1024), 256, 1023, 517, 255, 0, 48),
                                                   ((0, 0, 1920, 1080), 1024, 1919, 1079, 1023, 0, 140),
                                                   ((0, 0, 1920, 1080), 1024, 0, 0, 0, 0, 16),
                                                   ((0, 0, 3840, 2160), 4096, 2000, 1000, 4095, 100, 40)]:
        vals = ob.probe("sobol", *bounds, spp, px, py, sample, dim0, n).split()
        out["sobol"].append({"bounds": bounds, "spp": spp, "px": px, "py": py, "sample": sample, "dim0": dim0,
                             "values": vals})
    for (w, h, spp, px, py, n) in [(64, 64, 16, 3, 5, 16), (1920, 1080, 1024, 1900, 1000, 8)]:
        lines = ob.probe("camrays", *cam_args, w, h, spp, px, py, n).splitlines()
        out["camrays"].append({"res": [w, h], "spp": spp, "px": px, "py": py, "rays": [l.split() for l in lines]})
    consts = {}
    for line in ob.probe("consts").splitlines():
        k, *v = line.split()
        consts.setdefault(k, []).append(v)
    out["consts"] = consts
    json.dump(out, open(os.path.join(HERE, "probe.json"), "w"), indent=1)

    # ray/triangle + BVH answers from the real BVHAccel
    arr = scenes.SceneArrays(3000, materials=("matte",), soup_version=1, seed=99)
    rng = np.random.default_rng(5)
    n = 6000
    rays = np.zeros(n, dtype=abi.RAY_DTYPE)
    rays["o"] = rng.uniform(-1.2, 1.2, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d[: n // 2] /= np.linalg.norm(d[: n // 2], axis=1, keepdims=True)  # half unit, half unnormalised
    rays["d"] = d
    rays["t_max"] = np.inf
    rays["t_max"][n // 3: n // 2] = rng.uniform(0.05, 1.0, n // 2 - n // 3).astype(np.float32)
    # axis-aligned directions exercise the zero-component paths of the slab and watertight tests
    rays["d"][:30] = np.tile(np.eye(3, dtype=np.float32), (10, 1))
    tmp = "/tmp/golden_isect"
    os.makedirs(tmp, exist_ok=True)
    arr.vertices.tofile(os.path.join(tmp, "tris.f32"))
    rays.tofile(os.path.join(tmp, "rays.bin"))
    ob.probe("intersect", os.path.join(tmp, "tris.f32"), os.path.join(tmp, "rays.bin"), os.path.join(tmp, "out.bin"))
    res = np.fromfile(os.path.join(tmp, "out.bin"),
                      dtype=[("tri", "<i4"), ("t", "<f4"), ("p", "<f4", 3), ("n", "<f4", 3), ("perr", "<f4", 3),
                             ("occluded", "<i4")])
    np.save(os.path.join(HERE, "isect_rays.npy"), rays)
    np.save(os.path.join(HERE, "isect_ref.npy"), res)

    reference_renders(RENDERS)
    print("golden fixtures written to", HERE)


def reference_renders(names):
    """render_<name>.pfm of the reference for the given tests/render_cases.py RENDERS."""
    for name in names:
        nt, mats, w, h, spp, depth, strat, nl = RENDERS[name]
        ex = EXTRA.get(name, {})
        arr = scenes.SceneArrays(nt, materials=mats, soup_version=1, n_lights=nl, **ex.get("scene", {}))
        path = scenes.write_pbrt("/tmp/golden_render", "render_" + name, arr, w, h, spp, max_depth=depth,
                                 strategy=strat, **ex.get("camera", {}))
        ob.run_pbrt_ref(path, threads=1 if name.startswith("filter_") else None)
        os.replace(os.path.join("/tmp/golden_render", "render_%s.pfm" % name),
                   os.path.join(HERE, "render_%s.pfm" % name))


if __name__ == "__main__":
    if len(sys.argv) > 1:  # only the named render cases, e.g. one just added to tests/render_cases.py
        reference_renders(sys.argv[1:])
    else:
        main()
